"""Stage-2 RQTransformer (reference enhancing/modules/stage2/layers.py:306-547) -- the CPU part.

oracle/rq_oracle.py against the reference-generated goldens (tests/golden/rq_tiny.npz and ref_rq_class.npz, from
oracle/gen_golden_rq.py); etb.RQTransformer's construction, module tree and limits; its host logic with every C entry point
replaced by a torch stand-in written from include/b200vq.h; and the argument checks of the new entry points."""
import os
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import rq_oracle as R
from oracle.gen_golden_gpt import perturb
from oracle.gen_golden_rq import sd_digest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cfg(g):
    return {k[4:]: int(g[k]) for k in g.files if k.startswith("cfg.")}


def rebuilt_tiny(golden_dir):
    """rq_tiny.npz stores digests, not tables: rebuild the perturbed state dict from the seed with this package's class"""
    import enhancing_transformers_b200 as etb
    g = np.load(os.path.join(golden_dir, "rq_tiny.npz"))
    cfg = _cfg(g)
    torch.manual_seed(int(g["seed"]))
    model = etb.RQTransformer(**cfg)
    init = sd_digest(model.state_dict())
    perturb(model)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    # every test that uses the tables checks them against the reference's bits first
    assert init == str(g["init_sha256"]), "seeded construction differs from the reference's"
    assert sd_digest(sd) == str(g["sd_sha256"]), "rebuilt state dict differs from the reference's perturbed one"
    return g, cfg, sd, init


def _heads(cfg):
    return cfg["spatial_n_heads"], cfg["depth_n_heads"]


def _rel(a, b):
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


# ------------------------------------------------------------------------------------------- oracle and construction
def test_seeded_construction_gives_the_reference_state_dict_bit_for_bit(golden_dir):
    g, cfg, sd, init = rebuilt_tiny(golden_dir)
    assert init == str(g["init_sha256"])
    assert sd_digest(sd) == str(g["sd_sha256"])
    assert set(sd) == {k[6:] for k in g.files if k.startswith("shape.")}
    for k, v in sd.items():
        assert tuple(v.shape) == tuple(g["shape." + k]), k


def test_rq_oracle_matches_reference_golden(golden_dir):
    g, cfg, sd, _ = rebuilt_tiny(golden_dir)
    codes, conds = torch.from_numpy(g["codes"]), torch.from_numpy(g["conds"])
    sdg = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    loss, logits = R.rq_loss(sdg, codes, conds, *_heads(cfg))
    torch.testing.assert_close(logits.detach(), torch.from_numpy(g["logits"]), rtol=1e-5, atol=1e-6)
    assert abs(loss.item() - float(g["loss"])) < 1e-6
    loss.backward()
    names = [k[5:] for k in g.files if k.startswith("grad.")]
    assert set(names) == set(sd)
    for k in names:
        torch.testing.assert_close(sdg[k].grad, torch.from_numpy(g["grad." + k]), rtol=1e-4, atol=2e-7, msg=lambda m: f"{k}: {m}")


def test_rq_oracle_sampling_steps_match_reference_golden(golden_dir):
    g, cfg, sd, _ = rebuilt_tiny(golden_dir)
    sl = R.rq_sample_logits(sd, torch.from_numpy(g["conds"]), torch.from_numpy(g["sample_codes"]), *_heads(cfg))
    torch.testing.assert_close(sl, torch.from_numpy(g["sample_logits"]), rtol=1e-5, atol=1e-6)


def test_rq_oracle_matches_the_vendored_reference_class(golden_dir):
    """no biases, a 3-token prefix, a 64-wide spatial head and 32-wide depth heads, D = 3"""
    g = np.load(os.path.join(golden_dir, "ref_rq_class.npz"))
    cfg = _cfg(g)
    sd = {k[3:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("sd.")}
    out = R.rq_forward(sd, torch.from_numpy(g["codes"]), torch.from_numpy(g["conds"]), *_heads(cfg))
    torch.testing.assert_close(out, torch.from_numpy(g["logits"]), rtol=1e-5, atol=1e-6)


def test_module_tree_and_state_dict_match_reference(golden_dir):
    import enhancing_transformers_b200 as etb
    g = np.load(os.path.join(golden_dir, "ref_rq_class.npz"))
    cfg = _cfg(g)
    model = etb.RQTransformer(**cfg)
    sd = {k[3:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("sd.")}
    own = model.state_dict()
    assert set(own) == set(sd), set(own) ^ set(sd)
    model.load_state_dict(sd, strict=True)
    assert isinstance(model.spatial_transformer, torch.nn.Sequential) and isinstance(model.depth_transformer, torch.nn.Sequential)
    assert all(b.attn.short_seq for b in model.depth_transformer) and not any(b.attn.short_seq for b in model.spatial_transformer)
    assert model.depth_transformer[0].attn.ctx_len == 3 and model.depth_transformer[0].attn.cond_len == 0
    fresh = etb.RQTransformer(**cfg)
    assert fresh.pos_emb_depth.min().item() >= 0 and fresh.pos_emb_depth.max().item() < 1     # torch.rand, as in the reference
    assert fresh.ln_depth.weight.eq(1).all() and fresh.spatial_transformer[0].mlp.p0.weight.std().item() < 0.03
    gpt = etb.GPT(vocab_cond_size=10, vocab_img_size=64, embed_dim=64, cond_num_tokens=1, img_num_tokens=4, n_heads=2, n_layers=1)
    assert not gpt.blocks[0].attn.short_seq


@pytest.mark.parametrize("kw,match", [
    (dict(embed_dim=64, spatial_n_heads=4), "head size"),
    (dict(embed_dim=64, depth_n_heads=4), "head size"),
    (dict(embed_dim=4096, spatial_n_heads=64, depth_n_heads=64), "embed_dim"),
    (dict(embed_dim=96, spatial_n_heads=3, depth_n_heads=3), "embed_dim"),
    (dict(vocab_img_size=100), "vocab_img_size"),
    (dict(depth_num_tokens=1), "depth_num_tokens"),
    (dict(depth_num_tokens=17), "depth_num_tokens"),
])
def test_limits_reject_with_a_message(kw, match):
    import enhancing_transformers_b200 as etb
    cfg = dict(vocab_cond_size=10, vocab_img_size=64, embed_dim=64, cond_num_tokens=1, img_num_tokens=4, depth_num_tokens=4,
               spatial_n_heads=2, depth_n_heads=2, spatial_n_layers=1, depth_n_layers=1)
    cfg.update(kw)
    with pytest.raises(NotImplementedError, match=match):
        etb.RQTransformer(**cfg)


def test_patch_stage2_rebinds_rq_transformer():
    import enhancing_transformers_b200 as etb
    fake = types.ModuleType("fake_stage2_layers")
    fake.RQTransformer = object
    etb.patch_stage2(fake)
    assert fake.RQTransformer is etb.RQTransformer and fake.GPT is etb.GPT


# ------------------------------------------------------------------------------------------- host logic, kernels emulated
def _visible(D, cond, device=None):
    q = torch.arange(D, device=device).view(-1, 1)
    k = torch.arange(D, device=device).view(1, -1)
    return k <= torch.clamp(q, min=cond - 1)


def _short_attn(qkv, nseq, D, heads, hs, scale, cond):
    C = heads * hs
    t = qkv.view(nseq, D, 3, heads, hs).permute(2, 0, 3, 1, 4)           # [3, nseq, heads, D, hs]
    s = (t[0] @ t[1].transpose(-2, -1)) * scale
    s = s.masked_fill(~_visible(D, cond, qkv.device), float("-inf"))
    return (s.softmax(-1) @ t[2]).permute(0, 2, 1, 3).reshape(nseq * D, C)


def short_attention_fwd(qkv, nseq, D, heads, hs, scale, cond_len=0):
    return _short_attn(qkv, nseq, D, heads, hs, scale, cond_len)


def short_attention_bwd(qkv, dout, nseq, D, heads, hs, scale, cond_len=0):
    with torch.enable_grad():
        x = qkv.detach().clone().requires_grad_(True)
        (g,) = torch.autograd.grad(_short_attn(x, nseq, D, heads, hs, scale, cond_len), x, dout)
    return g


def _scan(rows):
    return rows.double().cumsum(-1).float()


def _rscan(rows):
    return rows.double().flip(-1).cumsum(-1).flip(-1).float()


def rq_embed_fwd(conds, codes, Wc, pos_c, Wi, pos_i):
    B, Tc = conds.shape
    C = Wi.shape[1]
    xc = Wc[conds] + pos_c.reshape(-1, C)
    xi = _scan(Wi[codes[..., -1]]) + pos_i.reshape(-1, C)
    return torch.cat([xc, xi], 1).reshape(-1, C)


def rq_embed_bwd(conds, codes, g, Vc, Vi, deterministic=False):
    B, Tc = conds.shape
    T = codes.shape[1]
    C = g.shape[-1]
    g3 = g.view(B, Tc + T, C)
    gWc = torch.zeros(Vc, C).index_add_(0, conds.reshape(-1), g3[:, :Tc].reshape(-1, C))
    gWi = _rscan(torch.zeros(Vi, C).index_add_(0, codes[..., -1].reshape(-1), g3[:, Tc:].reshape(-1, C)))
    return gWc, g3[:, :Tc].sum(0), gWi, g3[:, Tc:].sum(0)


def rq_depth_input_fwd(h, codes, Wi, pos_d):
    D = codes.shape[-1]
    C = Wi.shape[1]
    rest = _scan(Wi[codes.reshape(-1, D)[:, :-1]]) + pos_d.reshape(-1, C)
    return torch.cat([h.view(-1, 1, C), rest], 1).reshape(-1, C)


def rq_depth_input_bwd(codes, g, Vi, deterministic=False):
    D = codes.shape[-1]
    C = g.shape[-1]
    g3 = g.view(-1, D, C)
    gWi = _rscan(torch.zeros(Vi, C).index_add_(0, codes.reshape(-1, D)[:, :-1].reshape(-1), g3[:, 1:].reshape(-1, C)))
    return g3[:, 0].clone(), gWi, g3[:, 1:].sum(0)


def code_sum_embed(codes, n, Wi, pos):
    return Wi[codes[:, :n]].sum(1) + pos.view(1, -1)


RQ_NAMES = ("short_attention_fwd", "short_attention_bwd", "rq_embed_fwd", "rq_embed_bwd", "rq_depth_input_fwd", "rq_depth_input_bwd",
            "code_sum_embed")


def install_standins(monkeypatch):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import emulated_ops
    from enhancing_transformers_b200 import ops
    emulated_ops.install(monkeypatch)
    for n in RQ_NAMES:
        monkeypatch.setattr(ops, n, globals()[n])


@pytest.mark.parametrize("mode", ["parity", "tf32", "fp16"])
def test_host_logic_with_emulated_kernels(golden_dir, monkeypatch, mode):
    """stage2.py's RQTransformer wiring -- autograd Functions, row windows, depth sequences, KV caches, the sampler's step
    order -- with every C entry point replaced by its stand-in: the host side alone reproduces the reference golden"""
    import enhancing_transformers_b200 as etb
    install_standins(monkeypatch)
    g, cfg, sd, _ = rebuilt_tiny(golden_dir)
    prev = etb.set_precision(mode)
    try:
        model = etb.RQTransformer(**cfg)
        model.load_state_dict(sd, strict=True)
        codes, conds = torch.from_numpy(g["codes"]), torch.from_numpy(g["conds"])
        logits = model(codes, conds)
        loss = F.cross_entropy(logits.view(-1, logits.shape[-1]), codes.view(-1))
        loss.backward()
        half = mode == "fp16"
        assert _rel(logits.detach(), torch.from_numpy(g["logits"])) < (3e-3 if half else 1e-5)
        for name, p in model.named_parameters():
            want = torch.from_numpy(g["grad." + name])
            if name.endswith("attn.key.bias"):
                assert p.grad.abs().max().item() < 1e-4
                continue
            e = ((p.grad - want).norm() / want.norm().clamp_min(1e-12)).item()
            assert e < (1e-2 if half else 1e-4), (name, e)
        model.eval()
        torch.manual_seed(99)                                   # the seed the golden's sampler ran under
        s_logits, drawn = model.sample(conds, use_fp16=False)
        assert s_logits.shape == (codes.shape[0] * cfg["img_num_tokens"], cfg["depth_num_tokens"], cfg["vocab_img_size"])
        if not half:
            assert torch.equal(drawn, torch.from_numpy(g["sample_codes"]))
            assert _rel(s_logits, torch.from_numpy(g["sample_logits"])) < 1e-5
    finally:
        etb.set_precision(prev)


# ------------------------------------------------------------------------------------------- C entry points
def test_new_entry_points_reject_bad_arguments_before_touching_the_device():
    import enhancing_transformers_b200 as etb
    lib = etb._lib.lib()

    def err():
        return lib.b200vq_last_error().decode()
    fake = 256                                          # never dereferenced: every call below fails its argument checks
    for fn in (lib.b200vq_short_attention_fwd, lambda *a: lib.b200vq_short_attention_bwd(a[0], fake, *a[1:])):
        args = [fake, fake, 1000, 4, 8, 64, 0, 0.125, None]
        bad = list(args); bad[0] = None
        assert fn(*bad) < 0 and "null pointer" in err()
        for D in (0, 17):
            bad = list(args); bad[3] = D
            assert fn(*bad) < 0 and "1..16" in err()
        bad = list(args); bad[5] = 48
        assert fn(*bad) < 0 and "head size" in err()
        bad = list(args); bad[4] = 64                   # 64 * 64 > 2048
        assert fn(*bad) < 0 and "2048" in err()

    B, Tc, T, D, C, Vc, Vi = 2, 1, 16, 4, 64, 10, 256
    args = [fake] * 7 + [B, Tc, T, D, C, Vc, Vi, None]
    for name in ("b200vq_rq_embed_fwd", "b200vq_rq_embed_bwd"):
        fn = getattr(lib, name)
        bad = list(args); bad[1] = None
        assert fn(*bad) < 0 and "null pointer" in err()
        bad = list(args); bad[10] = 17
        assert fn(*bad) < 0 and "1..16" in err()
    ws = lib.b200vq_rq_embed_bwd_deterministic_workspace_bytes(B, Tc, T, D, C, Vc, Vi)
    assert ws >= B * T * 8
    dargs = [fake] * 7 + [B, Tc, T, D, C, Vc, Vi, fake, ws, None]
    bad = list(dargs); bad[14] = None
    assert lib.b200vq_rq_embed_bwd_deterministic(*bad) < 0 and "null pointer" in err()
    bad = list(dargs); bad[15] = ws - 1
    assert lib.b200vq_rq_embed_bwd_deterministic(*bad) < 0 and "workspace too small" in err()
    bad = list(dargs); bad[10] = 0
    assert lib.b200vq_rq_embed_bwd_deterministic(*bad) < 0 and "1..16" in err()

    nseq = B * T
    assert lib.b200vq_rq_depth_input_fwd(fake, None, fake, fake, fake, nseq, D, C, Vi, None) < 0 and "null pointer" in err()
    assert lib.b200vq_rq_depth_input_fwd(fake, fake, fake, fake, fake, nseq, 17, C, Vi, None) < 0 and "1..16" in err()
    assert lib.b200vq_rq_depth_input_bwd(fake, fake, None, fake, fake, nseq, D, C, Vi, None) < 0 and "null pointer" in err()
    assert lib.b200vq_rq_depth_input_bwd(fake, fake, fake, fake, fake, nseq, 0, C, Vi, None) < 0 and "1..16" in err()
    ws = lib.b200vq_rq_depth_input_bwd_deterministic_workspace_bytes(nseq, D, C, Vi)
    assert ws >= nseq * (D - 1) * 8
    dargs = [fake] * 5 + [nseq, D, C, Vi, fake, ws, None]
    bad = list(dargs); bad[9] = None
    assert lib.b200vq_rq_depth_input_bwd_deterministic(*bad) < 0 and "null pointer" in err()
    bad = list(dargs); bad[10] = ws - 1
    assert lib.b200vq_rq_depth_input_bwd_deterministic(*bad) < 0 and "workspace too small" in err()
    bad = list(dargs); bad[6] = 17
    assert lib.b200vq_rq_depth_input_bwd_deterministic(*bad) < 0 and "1..16" in err()
    assert lib.b200vq_code_sum_embed(None, 4, 4, fake, fake, fake, B, C, Vi, None) < 0 and "null pointer" in err()
    assert lib.b200vq_code_sum_embed(fake, 2, 4, fake, fake, fake, B, C, Vi, None) < 0 and "bad shape" in err()
