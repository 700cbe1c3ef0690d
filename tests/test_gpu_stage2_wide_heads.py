"""Stage-2 transformers with 96- and 128-wide attention heads on the GPU: the wide-head masked flash attention (forward, both
backward kernels and the delta kernel), the KV-cache step and the short-sequence depth attention against fp64 torch; `GPT` and
`RQTransformer` against the reference golden (tests/golden/ref_stage2_wide.npz) in every data path; and config 5's sequence
geometry at embed_dim 1024 with 8 heads of 128 against the fp64 oracle."""
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

from oracle import gpt_oracle as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_rq_transformer import _short_attn  # noqa: E402
from test_stage2_wide_heads import (check_against_golden, forced_gpt_steps, forced_rq_steps, rebuilt, rel,  # noqa: E402
                                    rel_l2)

pytestmark = pytest.mark.gpu
TOL = {"parity": (1e-4, 1e-3), "tf32": (1e-2, 3e-2), "fp16": (1e-2, 3e-2)}      # (logits, gradients), as for the 64-wide heads


def _mask(T, cond, device):
    m = torch.tril(torch.ones(T, T, device=device, dtype=torch.bool))
    m[:cond, :cond] = True
    return m


def _ref_attention(qkv, B, T, heads, hs, cond):
    q, k, v = (t.view(B, T, heads, hs).transpose(1, 2) for t in qkv.view(B, T, 3, heads * hs).unbind(2))
    att = (q @ k.transpose(-2, -1)) / math.sqrt(hs)
    att = att.masked_fill(~_mask(T, cond, qkv.device), float("-inf")).softmax(-1)
    return (att @ v).transpose(1, 2).reshape(B * T, heads * hs)


# ------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("exact", [True, False])
@pytest.mark.parametrize("hs", [96, 128])
@pytest.mark.parametrize("B,T,heads,cond", [(1, 1025, 2, 1), (2, 200, 2, 5), (1, 257, 3, 70), (2, 130, 1, 0), (1, 200, 2, 200),
                                            (3, 16, 2, 1), (1, 64, 1, 3)])
def test_attention_causal_fwd_bwd_wide(exact, hs, B, T, heads, cond):
    from enhancing_transformers_b200 import ops
    torch.manual_seed(T + cond + hs)
    qkv = torch.randn(B * T, 3 * heads * hs, device="cuda")
    dout = torch.randn(B * T, heads * hs, device="cuda")
    if not exact:
        qkv, dout = ops.round_tf32(qkv), ops.round_tf32(dout)
    scale = 1.0 / math.sqrt(hs)
    out, lse = ops.attention_causal_fwd(qkv, B, T, heads, hs, scale, cond, exact)
    dqkv = ops.attention_causal_bwd(qkv, out, lse, dout, B, T, heads, hs, scale, cond, exact)
    q64 = qkv.double().requires_grad_(True)
    ref = _ref_attention(q64, B, T, heads, hs, cond)
    ref.backward(dout.double())
    tol_o, tol_g = (2e-5, 5e-5) if exact else (2e-3, 4e-3)
    assert torch.isfinite(out).all() and torch.isfinite(dqkv).all()
    assert rel(out.double(), ref.detach()) < tol_o
    assert rel(dqkv.double(), q64.grad) < tol_g
    q, k, _ = (t.view(B, T, heads, hs).transpose(1, 2) for t in q64.detach().view(B, T, 3, heads * hs).unbind(2))
    s = ((q @ k.transpose(-2, -1)) * scale).masked_fill(~_mask(T, cond, "cuda"), float("-inf"))
    assert (lse.double().view(B, heads, T) - torch.logsumexp(s, -1)).abs().max().item() < (1e-4 if exact else 2e-3)
    # no atomics, every sum in an order fixed by the shape: a second launch gives the same bits
    out2, lse2 = ops.attention_causal_fwd(qkv, B, T, heads, hs, scale, cond, exact)
    dqkv2 = ops.attention_causal_bwd(qkv, out2, lse2, dout, B, T, heads, hs, scale, cond, exact)
    assert torch.equal(out, out2) and torch.equal(lse, lse2) and torch.equal(dqkv, dqkv2)


def test_attention_wide_tf32_round_out():
    """round_out on the single-pass path: the stored O and dqkv are tf32 values"""
    from enhancing_transformers_b200 import _lib, ops
    torch.manual_seed(3)
    B, T, heads, hs = 2, 150, 2, 128
    qkv = ops.round_tf32(torch.randn(B * T, 3 * heads * hs, device="cuda"))
    out = torch.empty(B * T, heads * hs, device="cuda")
    lse = torch.empty(B * heads * T, device="cuda")
    p = lambda t: t.data_ptr()   # noqa: E731
    lib = _lib.lib()
    stream = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.b200vq_attention_causal_fwd(p(qkv), p(out), p(lse), B, T, heads, hs, hs ** -0.5, 1, 0, 1, stream), "fwd")
    assert torch.equal(out, ops.round_tf32(out))
    dout = ops.round_tf32(torch.randn_like(out))
    dqkv, delta = torch.empty_like(qkv), torch.empty(B * heads * T, device="cuda")
    _lib.check(lib.b200vq_attention_causal_bwd(p(qkv), p(out), p(lse), p(dout), p(dqkv), p(delta), B, T, heads, hs, hs ** -0.5, 1, 0,
                                               1, stream), "bwd")
    assert torch.equal(dqkv, ops.round_tf32(dqkv))
    torch.testing.assert_close(delta.view(B, heads, T), (dout * out).view(B, T, heads, hs).sum(-1).transpose(1, 2), rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("hs", [96, 128])
@pytest.mark.parametrize("pos", [0, 17, 1024])
def test_decode_attention_wide(hs, pos):
    from enhancing_transformers_b200 import ops
    torch.manual_seed(pos + hs)
    heads = 3
    B, C, Tmax = 3, heads * hs, 1025
    ck, cv = torch.randn(B, Tmax, C, device="cuda"), torch.randn(B, Tmax, C, device="cuda")
    qkv = torch.randn(B, 3 * C, device="cuda")
    k_ref, v_ref = ck.clone(), cv.clone()
    k_ref[:, pos], v_ref[:, pos] = qkv[:, C:2 * C], qkv[:, 2 * C:]
    out = ops.decode_attention(qkv, ck, cv, heads, hs, pos, hs ** -0.5)
    assert torch.equal(ck, k_ref) and torch.equal(cv, v_ref)           # the step's key / value rows were appended
    q = qkv[:, :C].double().view(B, heads, 1, hs)
    K = k_ref[:, :pos + 1].double().view(B, pos + 1, heads, hs).transpose(1, 2)
    V = v_ref[:, :pos + 1].double().view(B, pos + 1, heads, hs).transpose(1, 2)
    ref = (((q @ K.transpose(-2, -1)) * hs ** -0.5).softmax(-1) @ V).reshape(B, C)
    assert rel(out.double(), ref) < 1e-5


@pytest.mark.parametrize("D", [2, 3, 8, 16])
@pytest.mark.parametrize("hs,heads", [(96, 1), (96, 4), (96, 21), (128, 3), (128, 16)])
def test_short_attention_wide_vs_fp64(D, hs, heads):
    from enhancing_transformers_b200 import ops
    torch.manual_seed(D * heads + hs)
    nseq = 41
    C = heads * hs
    qkv = torch.randn(nseq * D, 3 * C, device="cuda")
    dout = torch.randn(nseq * D, C, device="cuda")
    for cond in (0, 2):
        o = ops.short_attention_fwd(qkv, nseq, D, heads, hs, 1.0 / hs ** 0.5, cond)
        dq = ops.short_attention_bwd(qkv, dout, nseq, D, heads, hs, 1.0 / hs ** 0.5, cond)
        x = qkv.double().requires_grad_(True)
        o64 = _short_attn(x, nseq, D, heads, hs, 1.0 / hs ** 0.5, cond)
        (g64,) = torch.autograd.grad(o64, x, dout.double())
        assert rel(o.double(), o64.detach()) < 1e-5
        assert rel(dq.double(), g64) < 1e-5


# ------------------------------------------------------------------------------------------- models against the golden
@pytest.mark.parametrize("mode", ["parity", "tf32", "fp16"])
@pytest.mark.parametrize("name", ["gpt96", "gpt128"])
def test_gpt_wide_heads_match_reference_golden(golden_dir, mode, name):
    import enhancing_transformers_b200 as etb
    g, cfg, model = rebuilt(golden_dir, name)
    tl, tg = TOL[mode]
    prev = etb.set_precision(mode)
    try:
        model = model.cuda()
        codes, conds = torch.from_numpy(g[name + ".codes"]).cuda(), torch.from_numpy(g[name + ".conds"]).cuda()
        n0 = etb.ops.launch_count()
        logits = model(codes, conds)
        loss = F.cross_entropy(logits.view(-1, logits.shape[-1]), codes.view(-1))
        loss.backward()
        torch.cuda.synchronize()
        assert etb.ops.launch_count() - n0 > 30                      # the CUDA path ran
        # key.bias: zero in exact arithmetic, so its bound is absolute; one tf32 pass leaves rounding noise of ~3e-5 there at
        # these widths, within the bound of the host-logic test
        check_against_golden(g, name, model, logits, tl, tg, 1e-5 if mode == "parity" else 1e-4)
        assert abs(loss.item() - float(g[name + ".loss"])) < tl * abs(float(g[name + ".loss"])) * 10
    finally:
        etb.set_precision(prev)


@pytest.mark.parametrize("mode,tol", [("parity", 1e-4), ("fp16", 1e-2)])
@pytest.mark.parametrize("name", ["gpt96", "gpt128"])
def test_gpt_wide_heads_sampling_steps_match_reference_golden(golden_dir, mode, tol, name):
    import enhancing_transformers_b200 as etb
    g, cfg, model = rebuilt(golden_dir, name)
    prev = etb.set_precision(mode)
    try:
        model = model.cuda().eval()
        conds = torch.from_numpy(g[name + ".conds"]).cuda()
        codes = torch.from_numpy(g[name + ".sample_codes"]).cuda()
        steps = forced_gpt_steps(model, conds, codes).cpu()
        torch.manual_seed(0)
        s_logits, s_codes = model.sample(conds, top_k=7, top_p=0.9, softmax_temperature=0.8, use_fp16=False)
    finally:
        etb.set_precision(prev)
    assert rel(steps, torch.from_numpy(g[name + ".sample_logits"]).view_as(steps)) < tol
    T, V = cfg["img_num_tokens"], cfg["vocab_img_size"]
    assert s_codes.is_cuda and s_codes.shape == (2, T) and s_codes.min().item() >= 0 and s_codes.max().item() < V
    assert s_logits.shape == (2, T * V)


@pytest.mark.parametrize("mode", ["parity", "tf32", "fp16"])
def test_rq_wide_heads_match_reference_golden(golden_dir, mode):
    """128-wide spatial heads, 96-wide depth heads, at the tolerances of tests/test_gpu_rq_transformer.py"""
    import enhancing_transformers_b200 as etb
    g, cfg, model = rebuilt(golden_dir, "rq")
    tl, tg = TOL[mode]
    prev = etb.set_precision(mode)
    try:
        model = model.cuda()
        codes, conds = torch.from_numpy(g["rq.codes"]).cuda(), torch.from_numpy(g["rq.conds"]).cuda()
        logits = model(codes, conds)
        F.cross_entropy(logits.view(-1, logits.shape[-1]), codes.view(-1)).backward()
        check_against_golden(g, "rq", model, logits, tl, tg, 1e-3)
        model.eval()
        with torch.no_grad():
            sl = forced_rq_steps(model, conds, torch.from_numpy(g["rq.sample_codes"]).cuda())
        assert rel(sl.cpu(), torch.from_numpy(g["rq.sample_logits"])) < tl
        torch.manual_seed(0)
        s_logits, s_codes = model.sample(conds, top_k=7, use_fp16=False)
        assert s_codes.shape == (2, cfg["img_num_tokens"], cfg["depth_num_tokens"])
    finally:
        etb.set_precision(prev)


@pytest.mark.parametrize("mode,tol", [("parity", 1e-4), ("tf32", 1e-2), ("fp16", 1e-2)])
def test_gpt_config5_sequence_at_128_wide_heads_vs_fp64_oracle(mode, tol):
    """config 5's sequence geometry (1 class token + 32 x 32 codes = 1025 positions, 8192-entry vocabulary, 2 layers) at
    embed_dim 1024 with 8 heads of 128, against the oracle evaluated in fp64 on the GPU, with the bounds of
    test_stage2.py::test_gpt_base_shaped_sequence_vs_fp64_oracle"""
    import enhancing_transformers_b200 as etb
    cfg = dict(vocab_cond_size=1000, vocab_img_size=8192, embed_dim=1024, cond_num_tokens=1, img_num_tokens=1024, n_heads=8, n_layers=2)
    torch.manual_seed(11)
    model = etb.GPT(**cfg)
    with torch.no_grad():
        model.pos_emb_code.normal_(0, 0.1)
        model.pos_emb_cond.normal_(0, 0.1)
        for p in model.parameters():
            if p.dim() == 2:
                p.mul_(4.0)
    model = model.cuda()
    codes = torch.randint(0, 8192, (2, 1024), device="cuda")
    conds = torch.randint(0, 1000, (2, 1), device="cuda")
    prev = etb.set_precision(mode)
    try:
        logits = model(codes, conds)
        loss = F.cross_entropy(logits.view(-1, 8192), codes.view(-1))
        loss.backward()
    finally:
        etb.set_precision(prev)
    sd64 = {k: v.detach().double().requires_grad_(v.is_floating_point()) for k, v in model.state_dict().items()}
    loss64, logits64 = G.gpt_loss(sd64, codes, conds, 8)
    loss64.backward()
    r = rel(logits.detach().double(), logits64.detach())
    worst = max(rel_l2(p.grad.double(), sd64[n].grad) for n, p in model.named_parameters() if not n.endswith("attn.key.bias"))
    print(f"gpt 1025-token, 8 x 128 heads [{mode}] logits rel err {r:.2e}, worst grad rel-l2 {worst:.2e}")
    assert r < tol and worst < 30 * tol
