"""Stage-2 RQTransformer on the GPU: etb.RQTransformer against the reference golden and the fp64 oracle, the short-sequence
attention kernel against fp64 torch, the residual-code embedding kernels against torch, bit-reproducibility, and an end-to-end
RQ-VAE prior step."""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from oracle import rq_oracle as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_rq_transformer import _rel, _short_attn, rebuilt_tiny  # noqa: E402

pytestmark = pytest.mark.gpu
TOL = {"parity": (1e-4, 1e-3), "tf32": (1e-2, 3e-2), "fp16": (1e-2, 3e-2)}      # (logits, gradients), as for GPT


def _model(cfg, sd):
    import enhancing_transformers_b200 as etb
    m = etb.RQTransformer(**cfg)
    m.load_state_dict(sd, strict=True)
    return m.cuda()


def _forced_sample_logits(model, conds, codes):
    """the sampler's step functions with the codes forced: [B*T, D, vocab]"""
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


@pytest.mark.parametrize("mode", ["parity", "tf32", "fp16"])
def test_rq_transformer_matches_reference_golden(golden_dir, mode):
    import enhancing_transformers_b200 as etb
    g, cfg, sd, _ = rebuilt_tiny(golden_dir)
    tl, tg = TOL[mode]
    prev = etb.set_precision(mode)
    try:
        model = _model(cfg, sd)
        codes, conds = torch.from_numpy(g["codes"]).cuda(), torch.from_numpy(g["conds"]).cuda()
        logits = model(codes, conds)
        loss = F.cross_entropy(logits.view(-1, logits.shape[-1]), codes.view(-1))
        loss.backward()
        assert _rel(logits.detach().cpu(), torch.from_numpy(g["logits"])) < tl
        for name, p in model.named_parameters():
            want = torch.from_numpy(g["grad." + name])
            if name.endswith("attn.key.bias"):
                assert p.grad.abs().max().item() < 1e-3
                continue
            e = ((p.grad.cpu() - want).norm() / want.norm().clamp_min(1e-12)).item()
            assert e < tg, (name, e)
        model.eval()
        with torch.no_grad():
            sl = _forced_sample_logits(model, conds, torch.from_numpy(g["sample_codes"]).cuda())
        assert _rel(sl.cpu(), torch.from_numpy(g["sample_logits"])) < tl
    finally:
        etb.set_precision(prev)


@pytest.mark.parametrize("mode", ["parity", "tf32", "fp16"])
def test_realistic_shape_vs_fp64_oracle(mode):
    """B 2, T 1024, D 4, C 256, vocab 8192"""
    import enhancing_transformers_b200 as etb
    cfg = dict(vocab_cond_size=1000, vocab_img_size=8192, embed_dim=256, cond_num_tokens=1, img_num_tokens=1024, depth_num_tokens=4,
               spatial_n_heads=4, depth_n_heads=4, spatial_n_layers=2, depth_n_layers=2)
    torch.manual_seed(0)
    model = etb.RQTransformer(**cfg).cuda()
    gen = torch.Generator().manual_seed(1)
    codes = torch.randint(0, 8192, (2, 1024, 4), generator=gen).cuda()
    conds = torch.randint(0, 1000, (2, 1), generator=gen).cuda()
    tl, tg = TOL[mode]
    prev = etb.set_precision(mode)
    try:
        logits = model(codes, conds)
        F.cross_entropy(logits.view(-1, 8192), codes.view(-1)).backward()
    finally:
        etb.set_precision(prev)
    sd64 = {k: v.detach().double().requires_grad_(True) for k, v in model.state_dict().items()}
    loss64, ref = R.rq_loss(sd64, codes, conds, 4, 4)
    loss64.backward()
    assert _rel(logits.detach().double(), ref.detach()) < tl
    for name, p in model.named_parameters():
        want = sd64[name].grad
        if name.endswith("attn.key.bias"):
            continue
        e = ((p.grad.double() - want).norm() / want.norm().clamp_min(1e-30)).item()
        assert e < tg, (name, e)


# ------------------------------------------------------------------------------------------- short-sequence attention
def _ref64(qkv, nseq, D, heads, hs, cond, dout):
    x = qkv.double().requires_grad_(True)
    o = _short_attn(x, nseq, D, heads, hs, 1.0 / hs ** 0.5, cond)
    (g,) = torch.autograd.grad(o, x, dout.double())
    return o.detach(), g


@pytest.mark.parametrize("D", [1, 2, 4, 8, 16])
@pytest.mark.parametrize("hs", [32, 64])
@pytest.mark.parametrize("heads", [1, 3, 8])
def test_short_attention_vs_fp64(D, hs, heads):
    from enhancing_transformers_b200 import ops
    nseq = 37
    C = heads * hs
    qkv = torch.randn(nseq * D, 3 * C, device="cuda")
    dout = torch.randn(nseq * D, C, device="cuda")
    for cond in (0, 2):
        o = ops.short_attention_fwd(qkv, nseq, D, heads, hs, 1.0 / hs ** 0.5, cond)
        dq = ops.short_attention_bwd(qkv, dout, nseq, D, heads, hs, 1.0 / hs ** 0.5, cond)
        o64, g64 = _ref64(qkv, nseq, D, heads, hs, cond, dout)
        assert _rel(o.double(), o64) < 1e-5
        assert _rel(dq.double(), g64) < 1e-5


def test_short_attention_beyond_the_grid_z_limit():
    """B' > 65 535 sequences (a batch of 64 images of 1024 positions); repeated calls give the same bits"""
    from enhancing_transformers_b200 import ops
    nseq, D, heads, hs = 65536 + 77, 4, 2, 32
    C = heads * hs
    qkv = torch.randn(nseq * D, 3 * C, device="cuda")
    dout = torch.randn(nseq * D, C, device="cuda")
    o = ops.short_attention_fwd(qkv, nseq, D, heads, hs, 1.0 / hs ** 0.5)
    dq = ops.short_attention_bwd(qkv, dout, nseq, D, heads, hs, 1.0 / hs ** 0.5)
    o64, g64 = _ref64(qkv, nseq, D, heads, hs, 0, dout)
    assert _rel(o.double(), o64) < 1e-5 and _rel(dq.double(), g64) < 1e-5
    assert torch.equal(o, ops.short_attention_fwd(qkv, nseq, D, heads, hs, 1.0 / hs ** 0.5))
    assert torch.equal(dq, ops.short_attention_bwd(qkv, dout, nseq, D, heads, hs, 1.0 / hs ** 0.5))


def test_short_attention_sequences_do_not_leak():
    from enhancing_transformers_b200 import ops
    nseq, D, heads, hs = 301, 4, 4, 64
    C = heads * hs
    qkv = torch.randn(nseq, D, 3 * C, device="cuda")
    dout = torch.randn(nseq, D, C, device="cuda")
    o = ops.short_attention_fwd(qkv.view(-1, 3 * C), nseq, D, heads, hs, 0.125)
    dq = ops.short_attention_bwd(qkv.view(-1, 3 * C), dout.view(-1, C), nseq, D, heads, hs, 0.125)
    qkv2, dout2 = qkv.clone(), dout.clone()
    qkv2[1::2] *= 100
    dout2[1::2] *= 100
    o2 = ops.short_attention_fwd(qkv2.view(-1, 3 * C), nseq, D, heads, hs, 0.125).view(nseq, D, C)
    dq2 = ops.short_attention_bwd(qkv2.view(-1, 3 * C), dout2.view(-1, C), nseq, D, heads, hs, 0.125).view(nseq, D, 3 * C)
    assert torch.equal(o.view(nseq, D, C)[0::2], o2[0::2])
    assert torch.equal(dq.view(nseq, D, 3 * C)[0::2], dq2[0::2])


# ------------------------------------------------------------------------------------------- embedding kernels
def _embed_case(B=4, Tc=2, T=64, D=4, C=1024, Vc=10, Vi=512):
    gen = torch.Generator().manual_seed(3)
    Wc, Wi = torch.randn(Vc, C, generator=gen) * 0.02, torch.randn(Vi, C, generator=gen) * 0.02
    pc, pi, pd = torch.rand(Tc, C, generator=gen), torch.rand(T, C, generator=gen), torch.rand(D - 1, C, generator=gen)
    conds = torch.randint(0, Vc, (B, Tc), generator=gen)
    codes = torch.randint(0, Vi, (B, T, D), generator=gen)
    codes[0, :, :] = 7                                          # one id hit by many entries
    return conds, codes, Wc, pc, Wi, pi, pd


def test_embedding_forward_rows_equal_the_reference_formula_bit_for_bit():
    from enhancing_transformers_b200 import ops
    conds, codes, Wc, pc, Wi, pi, pd = _embed_case()
    B, T, D = codes.shape
    C = Wi.shape[1]
    x = ops.rq_embed_fwd(conds.cuda(), codes.cuda(), Wc.cuda(), pc.cuda(), Wi.cuda(), pi.cuda()).cpu().view(B, -1, C)
    cs = Wi[codes].cumsum(-1)                                   # layers.py:375-378, torch on the CPU
    assert torch.equal(x[:, :2], Wc[conds] + pc)
    assert torch.equal(x[:, 2:], cs[..., -1, :] + pi)
    h = torch.randn(B * T, C)
    v = ops.rq_depth_input_fwd(h.cuda(), codes.cuda(), Wi.cuda(), pd.cuda()).cpu().view(B, T, D, C)
    assert torch.equal(v[:, :, 0], h.view(B, T, C))
    assert torch.equal(v[:, :, 1:], cs[..., :-1, :] + pd)


def test_embedding_backward_vs_fp64_and_deterministic_path():
    from enhancing_transformers_b200 import ops
    conds, codes, Wc, pc, Wi, pi, pd = _embed_case()
    B, T, D = codes.shape
    C, Vc, Vi = Wi.shape[1], Wc.shape[0], Wi.shape[0]
    g_x = torch.randn(B * (2 + T), C)
    g_v = torch.randn(B * T * D, C)
    W64 = {n: t.double().requires_grad_(True) for n, t in dict(Wc=Wc, pc=pc, Wi=Wi, pi=pi, pd=pd).items()}
    h64 = torch.zeros(B * T, C, dtype=torch.float64, requires_grad=True)
    e = W64["Wi"][codes].cumsum(-1)
    x64 = torch.cat([W64["Wc"][conds] + W64["pc"], e[..., -1, :] + W64["pi"]], 1).view(-1, C)
    v64 = torch.cat([h64.view(B, T, 1, C), e[..., :-1, :] + W64["pd"]], 2).view(-1, C)
    ((x64 * g_x.double()).sum() + (v64 * g_v.double()).sum()).backward()
    cu = lambda t: t.cuda()                                     # noqa: E731
    gx, gv = cu(g_x), cu(g_v)
    results = {}
    for det in (False, True):
        gWc, gpc, gWi1, gpi = ops.rq_embed_bwd(cu(conds), cu(codes), gx, Vc, Vi, deterministic=det)
        gh, gWi2, gpd = ops.rq_depth_input_bwd(cu(codes), gv, Vi, deterministic=det)
        results[det] = (gWc, gpc, gWi1, gpi, gh, gWi2, gpd)
        got = dict(Wc=gWc, pc=gpc, Wi=gWi1 + gWi2, pi=gpi, pd=gpd)
        for n, t in got.items():
            assert _rel(t.double().cpu(), W64[n].grad) < 1e-5, (det, n)
        assert torch.equal(gh.cpu(), g_v.view(B, T, D, C)[:, :, 0].reshape(-1, C))
    # the deterministic path: the same bits on every call, and under an SM limit of 8
    again = []
    for limit in (0, 8):
        ops.set_sm_limit(limit)
        try:
            again.append(ops.rq_embed_bwd(cu(conds), cu(codes), gx, Vc, Vi, deterministic=True)
                         + ops.rq_depth_input_bwd(cu(codes), gv, Vi, deterministic=True))
        finally:
            ops.set_sm_limit(0)
    for a, b in zip(results[True], again[0]):
        assert torch.equal(a, b)
    for a, b in zip(again[0], again[1]):
        assert torch.equal(a, b)


def test_code_sum_embed():
    from enhancing_transformers_b200 import ops
    Wi = torch.randn(300, 128, device="cuda")
    codes = torch.randint(0, 300, (5, 40), device="cuda")
    pos = torch.rand(128, device="cuda")
    for n in (1, 3, 4):
        got = ops.code_sum_embed(codes[:, 8:8 + n], n, Wi, pos)
        torch.testing.assert_close(got, Wi[codes[:, 8:8 + n]].sum(1) + pos, rtol=1e-6, atol=1e-6)


# ------------------------------------------------------------------------------------------- whole module
_DET_SCRIPT = r"""
import hashlib, torch, torch.nn.functional as F
import enhancing_transformers_b200 as etb
torch.manual_seed(0)
m = etb.RQTransformer(vocab_cond_size=10, vocab_img_size=256, embed_dim=128, cond_num_tokens=1, img_num_tokens=64,
                      depth_num_tokens=4, spatial_n_heads=2, depth_n_heads=4, spatial_n_layers=2, depth_n_layers=2).cuda()
codes = torch.randint(0, 16, (8, 64, 4), device="cuda")        # few ids: many entries per embedding row
conds = torch.randint(0, 10, (8, 1), device="cuda")
F.cross_entropy(m(codes, conds).view(-1, 256), codes.view(-1)).backward()
h = hashlib.sha256()
for n, p in m.named_parameters():
    h.update(p.grad.cpu().numpy().tobytes())
print(h.hexdigest())
"""


def test_deterministic_switch_gives_identical_gradient_bits():
    env = dict(os.environ, B200VQ_DETERMINISTIC="1", PYTHONPATH=ROOT)
    outs = [subprocess.run([sys.executable, "-c", _DET_SCRIPT], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
            for _ in range(2)]
    for o in outs:
        assert o.returncode == 0, o.stderr[-2000:]
    assert outs[0].stdout.split()[-1] == outs[1].stdout.split()[-1]


class _Stage1(torch.nn.Module):
    """The stage-1 surface an RQ prior is trained against: the reference ViTVQ's encode_codes / decode / decode_codes
    (vitvqgan.py:68-90) restated over this package's modules.  ViTVQ itself is a LightningModule of the reference package
    and cannot be built without it; these methods run the same operations on the same attributes, so a code-shape
    mismatch between the quantiser, the prior and decode_codes shows up here as it would there."""

    def __init__(self):
        import enhancing_transformers_b200 as etb
        super().__init__()
        self.encoder = etb.ViTEncoder(32, 8, dim=64, depth=1, heads=2, mlp_dim=128, dim_head=32)
        self.pre_quant = etb.QuantLinear(64, 32)
        self.quantizer = etb.VectorQuantizer(embed_dim=32, n_embed=128, use_residual=True, num_quantizers=4)
        self.post_quant = etb.QuantLinear(32, 64)
        self.decoder = etb.ViTDecoder(32, 8, dim=64, depth=1, heads=2, mlp_dim=128, dim_head=32)

    def encode_codes(self, x):                                  # vitvqgan.py:74-79
        _, _, codes = self.quantizer(self.pre_quant(self.encoder(x)))
        return codes

    def decode(self, quant):                                    # vitvqgan.py:68-72
        return self.decoder(self.post_quant(quant))

    def decode_codes(self, code):                               # vitvqgan.py:81-90
        quant = self.quantizer.norm(self.quantizer.embedding(code))
        if self.quantizer.use_residual:
            quant = quant.sum(-2)
        return self.decode(quant)


def test_end_to_end_rq4_prior():
    """RQ4 stage 1 -> encode_codes -> RQTransformer cross-entropy and backward (CondTransformer.shared_step,
    stage2/transformer.py:107-118); sample -> decode_codes (transformer.py:79-95, code_shape None) gives images"""
    import enhancing_transformers_b200 as etb
    torch.manual_seed(0)
    stage1 = _Stage1().cuda()
    img = torch.rand(3, 3, 32, 32, device="cuda")
    with torch.no_grad():
        codes = stage1.encode_codes(img).detach()
    assert codes.shape == (3, 16, 4)                            # [B, positions, num_quantizers], fed to the prior as is
    prior = etb.RQTransformer(vocab_cond_size=5, vocab_img_size=128, embed_dim=64, cond_num_tokens=1, img_num_tokens=16,
                              depth_num_tokens=4, spatial_n_heads=2, depth_n_heads=2, spatial_n_layers=1, depth_n_layers=1).cuda()
    conds = torch.zeros(3, 1, dtype=torch.int64, device="cuda")
    logits = prior(codes, conds)
    loss = F.cross_entropy(logits.view(-1, logits.shape[-1]), codes.view(-1))
    loss.backward()
    assert torch.isfinite(loss) and all(p.grad is not None and torch.isfinite(p.grad).all() for p in prior.parameters())
    prior.eval()
    s_logits, s_codes = prior.sample(conds.view(conds.shape[0], -1), top_k=20)
    assert s_logits.shape == (48, 4, 128) and s_codes.shape == (3, 16, 4)
    with torch.no_grad():
        pixels = stage1.decode_codes(s_codes).clamp(0, 1)
        fast = stage1.decode(stage1.quantizer.embed_codes(s_codes))     # the package's one-kernel decode_codes path
    assert pixels.shape == (3, 3, 32, 32) and torch.isfinite(pixels).all()
    torch.testing.assert_close(fast.clamp(0, 1), pixels, rtol=1e-4, atol=1e-4)


def test_rq_embed_backward_without_cond_rows_zeroes_the_cond_table():
    from enhancing_transformers_b200 import ops
    conds = torch.zeros(2, 0, dtype=torch.int64, device="cuda")
    codes = torch.randint(0, 64, (2, 8, 4), device="cuda")
    g = torch.randn(2 * 8, 64, device="cuda")
    for det in (False, True):
        gWc = ops.rq_embed_bwd(conds, codes, g, 10, 64, deterministic=det)[0]
        assert gWc.shape == (10, 64) and gWc.eq(0).all()


def test_short_attention_under_an_sm_limit_gives_the_same_bits():
    from enhancing_transformers_b200 import ops
    nseq, D, heads, hs = 5000, 4, 4, 64
    qkv = torch.randn(nseq * D, 3 * heads * hs, device="cuda")
    dout = torch.randn(nseq * D, heads * hs, device="cuda")
    o = ops.short_attention_fwd(qkv, nseq, D, heads, hs, 0.125)
    dq = ops.short_attention_bwd(qkv, dout, nseq, D, heads, hs, 0.125)
    ops.set_sm_limit(8)
    try:
        assert torch.equal(o, ops.short_attention_fwd(qkv, nseq, D, heads, hs, 0.125))
        assert torch.equal(dq, ops.short_attention_bwd(qkv, dout, nseq, D, heads, hs, 0.125))
    finally:
        ops.set_sm_limit(0)
