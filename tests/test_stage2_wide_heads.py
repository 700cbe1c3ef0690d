"""Stage-2 transformers with 96- and 128-wide attention heads -- the CPU part.

`GPT` and `RQTransformer` at head sizes 96 and 128: seeded construction and state dict against the reference classes' (digests in
tests/golden/ref_stage2_wide.npz, from oracle/gen_golden_stage2_wide.py), the head sizes that stay rejected, the C entry points'
argument checks at the new sizes, and the host logic in all three data paths with every C entry point replaced by a torch
stand-in (tests/emulated_ops.py, and the RQ stand-ins of tests/test_rq_transformer.py) against the reference golden."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle.gen_golden_gpt import perturb
from oracle.gen_golden_rq import sd_digest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = ("gpt96", "gpt128", "rq")


def wide_golden(golden_dir):
    return np.load(os.path.join(golden_dir, "ref_stage2_wide.npz"))


def case_cfg(g, name):
    p = name + ".cfg."
    return {k[len(p):]: int(g[k]) for k in g.files if k.startswith(p)}


def rebuilt(golden_dir, name):
    """-> (golden, cfg, model): this package's class built from the golden's seed and perturbed as the reference's was; its
    state dict is checked against the reference's digests (keys, shapes and every bit) before it is returned"""
    import enhancing_transformers_b200 as etb
    g = wide_golden(golden_dir)
    cfg = case_cfg(g, name)
    torch.manual_seed(int(g[name + ".seed"]))
    model = (etb.RQTransformer if name == "rq" else etb.GPT)(**cfg)
    assert sd_digest(model.state_dict()) == str(g[name + ".init_sha256"]), f"{name}: seeded construction differs from the reference's"
    perturb(model)
    assert sd_digest(model.state_dict()) == str(g[name + ".sd_sha256"]), f"{name}: perturbed state dict differs from the reference's"
    return g, cfg, model


def golden_grad(g, name, pname, grad):
    """(mine, reference) for one parameter gradient: whole, or at the stored sample positions"""
    want = torch.from_numpy(g[f"{name}.grad.{pname}"])
    key = f"{name}.grad_idx.{pname}"
    if key in g.files:
        return grad.reshape(-1)[torch.from_numpy(g[key])], want
    return grad, want


def rel(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


def rel_l2(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def head_sizes(cfg):
    if "n_heads" in cfg:
        return {cfg["embed_dim"] // cfg["n_heads"]}
    return {cfg["embed_dim"] // cfg["spatial_n_heads"], cfg["embed_dim"] // cfg["depth_n_heads"]}


# ------------------------------------------------------------------------------------------- construction and limits
@pytest.mark.parametrize("name", CASES)
def test_seeded_construction_and_state_dict_match_the_reference(golden_dir, name):
    g, cfg, model = rebuilt(golden_dir, name)
    assert head_sizes(cfg) <= {96, 128} and head_sizes(cfg) & {96, 128}
    own = model.state_dict()
    assert model.load_state_dict({k: v.clone() for k, v in own.items()}, strict=True)
    kinds = {type(m) for m in model.modules()}
    assert {torch.nn.Linear, torch.nn.LayerNorm, torch.nn.Embedding} <= kinds
    blocks = [model.blocks] if name != "rq" else [model.spatial_transformer, model.depth_transformer]
    for stack in blocks:
        assert isinstance(stack, torch.nn.Sequential)
        for blk in stack:
            C = cfg["embed_dim"]
            assert blk.attn.query.weight.shape == (C, C) and blk.mlp.p0.weight.shape == (4 * C, C)
    if name == "rq":
        assert model.spatial_transformer[0].attn.n_heads == 3 and model.depth_transformer[0].attn.n_heads == 4
        assert all(b.attn.short_seq for b in model.depth_transformer)
    # every stored gradient names a parameter of the replacement, and every parameter has one
    assert {k[len(name) + 6:] for k in g.files if k.startswith(name + ".grad.")} == {n for n, _ in model.named_parameters()}


@pytest.mark.parametrize("hs", [48, 160, 192, 256, 384])
def test_head_sizes_without_a_kernel_are_rejected_with_a_message(hs):
    import enhancing_transformers_b200 as etb
    heads = 4 if hs == 48 else 2
    C = hs * heads                                       # a multiple of 64 <= 768: only the head size is at fault
    with pytest.raises(NotImplementedError, match="head size"):
        etb.GPT(vocab_cond_size=10, vocab_img_size=64, embed_dim=C, cond_num_tokens=1, img_num_tokens=4, n_heads=heads, n_layers=1)
    base = dict(vocab_cond_size=10, vocab_img_size=64, embed_dim=C, cond_num_tokens=1, img_num_tokens=4, depth_num_tokens=4,
                spatial_n_layers=1, depth_n_layers=1)
    ok = C // 128 if C % 128 == 0 else C // 96 if C % 96 == 0 else C // 64
    for sp, dp in ((heads, ok), (ok, heads)):
        with pytest.raises(NotImplementedError, match="head size"):
            etb.RQTransformer(spatial_n_heads=sp, depth_n_heads=dp, **base)


def test_wide_heads_keep_the_embed_dim_limits():
    import enhancing_transformers_b200 as etb
    with pytest.raises(NotImplementedError, match="embed_dim"):          # 128-wide heads, but embed_dim > 2048
        etb.GPT(vocab_cond_size=10, vocab_img_size=64, embed_dim=4096, cond_num_tokens=1, img_num_tokens=4, n_heads=32, n_layers=1)
    with pytest.raises(NotImplementedError, match="embed_dim"):          # 96-wide heads, an odd count: not a multiple of 64
        etb.GPT(vocab_cond_size=10, vocab_img_size=64, embed_dim=288, cond_num_tokens=1, img_num_tokens=4, n_heads=3, n_layers=1)
    for C, heads in ((192, 2), (256, 2), (1024, 8), (384, 4)):
        etb.GPT(vocab_cond_size=4, vocab_img_size=64, embed_dim=C, cond_num_tokens=1, img_num_tokens=2, n_heads=heads, n_layers=1)


def test_c_abi_checks_wide_head_sizes_before_touching_the_device():
    import enhancing_transformers_b200 as etb
    lib = etb._lib.lib()

    def err():
        return lib.b200vq_last_error().decode()
    for hs in (48, 160, 192, 256, 384):
        assert lib.b200vq_attention_causal_fwd(None, None, None, 1, 16, 2, hs, 0.1, 1, 1, 0, None) < 0 and "head size" in err()
        assert lib.b200vq_attention_causal_bwd(None, None, None, None, None, None, 1, 16, 2, hs, 0.1, 1, 0, 0, None) < 0
        assert "head size" in err()
        assert lib.b200vq_decode_attention(None, None, None, None, 2, 2, hs, 10, 3, 0.1, None) < 0 and "head size" in err()
        for fn in (lib.b200vq_short_attention_fwd, lambda *a: lib.b200vq_short_attention_bwd(a[0], 256, *a[1:])):
            assert fn(256, 256, 1000, 4, 2, hs, 0, 0.1, None) < 0 and "head size" in err()
    # 96 and 128 pass the head-size check and stop at the next one, still before any launch
    for hs in (96, 128):
        assert lib.b200vq_attention_causal_fwd(None, None, None, 1, 16, 2, hs, 0.1, 17, 1, 0, None) < 0 and "cond_len" in err()
        assert lib.b200vq_attention_causal_bwd(None, None, None, None, None, None, 0, 16, 2, hs, 0.1, 1, 0, 0, None) < 0
        assert "empty" in err()
        assert lib.b200vq_decode_attention(None, None, None, None, 2, 2, hs, 10, 10, 0.1, None) < 0 and "position" in err()
        for fn in (lib.b200vq_short_attention_fwd, lambda *a: lib.b200vq_short_attention_bwd(a[0], 256, *a[1:])):
            assert fn(256, 256, 1000, 17, 2, hs, 0, 0.1, None) < 0 and "1..16" in err()
            assert fn(256, 256, 1000, 4, 2048 // hs + 1, hs, 0, 0.1, None) < 0 and "2048" in err()
    # the stage-1 cores keep their head sizes and messages
    assert lib.b200vq_attention_fwd(None, None, 0, None, 1, 16, 2, 128, 0.1, 0, None) < 0 and "32 or 64" in err()
    assert lib.b200vq_attention_exact_fwd(None, None, None, 1, 16, 2, 96, 0.1, None) < 0 and "32 or 64" in err()
    assert lib.b200vq_attention_f16_fwd(None, None, None, 1, 16, 2, 128, 0.1, None) < 0 and "64" in err()


# ------------------------------------------------------------------------------------------- host logic, kernels emulated
def install_standins(monkeypatch):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import test_rq_transformer
    test_rq_transformer.install_standins(monkeypatch)    # tests/emulated_ops.py plus the RQ entry points


def forced_gpt_steps(model, conds, codes):
    past, got = None, []
    for i in range(codes.shape[1]):
        lg, past = model.sample_step(None if i == 0 else codes[:, i - 1:i], conds,
                                     None if i == 0 else model.pos_emb_code[:, i - 1:i, :], False, past)
        got.append(lg)
    return torch.stack(got, 1)


def forced_rq_steps(model, conds, codes):
    """the RQ sampler's step functions with the codes forced: [B*T, D, vocab]"""
    B, T, D = codes.shape
    out, past, depth_past = [], None, None
    for t in range(T):
        prev = None if t == 0 else codes[:, t - 1].contiguous()
        pos = None if t == 0 else model.pos_emb_code[:, t - 1:t, :]
        hidden, past = model.sample_spatial_step(prev, conds, pos, False, past)
        for d in range(D):
            cur = None if d == 0 else codes[:, t, :d].contiguous()
            pos_d = None if d == 0 else model.pos_emb_depth[:, d - 1:d, :]
            lg, depth_past = model.sample_depth_step(cur, hidden, pos_d, False, depth_past)
            out.append(lg)
    return torch.stack(out, 1).view(B * T, D, -1)


def check_against_golden(g, name, model, logits, tl, tg, key_bias_tol):
    """logits (max-relative) and every parameter gradient (relative l2) of `model` after backward"""
    assert rel(logits.detach().cpu(), torch.from_numpy(g[name + ".logits"])) < tl
    for pname, p in model.named_parameters():
        assert p.grad is not None, pname
        mine, want = golden_grad(g, name, pname, p.grad.detach().cpu())
        if pname.endswith("attn.key.bias"):               # exactly zero in exact arithmetic (softmax shift invariance)
            assert mine.abs().max().item() < key_bias_tol, pname
            continue
        e = rel_l2(mine, want)
        assert e < tg, (name, pname, e)


@pytest.mark.parametrize("mode", ["parity", "tf32", "fp16"])
@pytest.mark.parametrize("name", ["gpt96", "gpt128"])
def test_gpt_host_logic_at_wide_heads_with_emulated_kernels(golden_dir, monkeypatch, mode, name):
    """stage2.py's GPT wiring at 96- and 128-wide heads with every C entry point emulated, against the reference golden at the
    tolerances of test_stage2.py::test_gpt_host_logic_with_emulated_kernels"""
    import enhancing_transformers_b200 as etb
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import emulated_ops
    emulated_ops.install(monkeypatch)
    g, cfg, model = rebuilt(golden_dir, name)
    prev = etb.set_precision(mode)
    try:
        codes, conds = torch.from_numpy(g[name + ".codes"]), torch.from_numpy(g[name + ".conds"])
        logits = model(codes, conds)
        F.cross_entropy(logits.view(-1, logits.shape[-1]), codes.view(-1)).backward()
        half = mode == "fp16"
        check_against_golden(g, name, model, logits, 3e-3 if half else 1e-5, 1e-2 if half else 1e-4, 1e-4)
        model.eval()
        s_codes = torch.from_numpy(g[name + ".sample_codes"])
        steps = forced_gpt_steps(model, conds, s_codes)
        assert rel(steps, torch.from_numpy(g[name + ".sample_logits"]).view_as(steps)) < (3e-3 if half else 1e-5)
        torch.manual_seed(99)
        _, drawn = model.sample(conds, use_fp16=False)
        torch.manual_seed(123)
        d_logits, d_codes = model.sample(conds, use_fp16=False, top_k=7, top_p=0.9, softmax_temperature=0.8)
        if not half:
            assert torch.equal(drawn, s_codes)
            assert torch.equal(d_codes, torch.from_numpy(g[name + ".draw_codes"]))
            want = torch.from_numpy(g[name + ".draw_logits"])
            finite = torch.isfinite(want)
            assert torch.equal(finite, torch.isfinite(d_logits))
            torch.testing.assert_close(d_logits[finite], want[finite], rtol=1e-4, atol=1e-5)
    finally:
        etb.set_precision(prev)


@pytest.mark.parametrize("mode", ["parity", "tf32", "fp16"])
def test_rq_host_logic_at_wide_heads_with_emulated_kernels(golden_dir, monkeypatch, mode):
    """RQTransformer with 128-wide spatial and 96-wide depth heads, every C entry point emulated, against the reference golden at
    the tolerances of test_rq_transformer.py::test_host_logic_with_emulated_kernels"""
    import enhancing_transformers_b200 as etb
    install_standins(monkeypatch)
    g, cfg, model = rebuilt(golden_dir, "rq")
    prev = etb.set_precision(mode)
    try:
        codes, conds = torch.from_numpy(g["rq.codes"]), torch.from_numpy(g["rq.conds"])
        logits = model(codes, conds)
        F.cross_entropy(logits.view(-1, logits.shape[-1]), codes.view(-1)).backward()
        half = mode == "fp16"
        check_against_golden(g, "rq", model, logits, 3e-3 if half else 1e-5, 1e-2 if half else 1e-4, 1e-4)
        model.eval()
        with torch.no_grad():
            steps = forced_rq_steps(model, conds, torch.from_numpy(g["rq.sample_codes"]))
        assert rel(steps, torch.from_numpy(g["rq.sample_logits"])) < (3e-3 if half else 1e-5)
        torch.manual_seed(99)
        s_logits, drawn = model.sample(conds, use_fp16=False)
        assert s_logits.shape == (codes.shape[0] * cfg["img_num_tokens"], cfg["depth_num_tokens"], cfg["vocab_img_size"])
        torch.manual_seed(123)
        _, d_codes = model.sample(conds, use_fp16=False, top_k=7, top_p=0.9, softmax_temperature=0.8)
        if not half:
            assert torch.equal(drawn, torch.from_numpy(g["rq.sample_codes"]))
            assert rel(s_logits, torch.from_numpy(g["rq.sample_logits"])) < 1e-5
            assert torch.equal(d_codes, torch.from_numpy(g["rq.draw_codes"]))
    finally:
        etb.set_precision(prev)
