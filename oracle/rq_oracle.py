"""TEST INFRASTRUCTURE ONLY -- CPU / fp64 restatement of the reference's stage-2 ``RQTransformer``
(reference enhancing/modules/stage2/layers.py:306-547), the checker for ``enhancing_transformers_b200.stage2.RQTransformer``.
Nothing in the product package imports this file.

Pure functions over a flat state dict (the reference's own ``RQTransformer.state_dict()`` keys), in plain torch ops so that
they run in fp32 on the CPU and in fp64 on a GPU.  The blocks are gpt_oracle's (the same ``Block`` class, layers.py:112-143).
Pinned by ``tests/golden/rq_tiny.npz`` (oracle/gen_golden_rq.py, from the unmodified reference class) and
``tests/golden/ref_rq_class.npz`` (the vendored class in oracle/_ref)."""
import math

import torch
import torch.nn.functional as F

from oracle.gpt_oracle import _ln, attention, ffn, time_mix


def n_layers_of(sd, prefix):
    return 1 + max(int(k.split(".")[1]) for k in sd if k.startswith(prefix + "."))


def block(sd, p, x, n_heads, cond_len):
    """Block.forward, layers.py:132-136"""
    a, _, _ = attention(sd, p + "attn.", _ln(x, sd[p + "ln1.weight"], sd[p + "ln1.bias"]), n_heads, cond_len)
    x = x + a
    return x + ffn(sd, p + "mlp.", _ln(x, sd[p + "ln2.weight"], sd[p + "ln2.bias"]))


def rq_forward(sd, codes, conds, spatial_heads, depth_heads):
    """RQTransformer.forward, layers.py:370-395: codes [B, T, D], conds [B, Tc] -> logits [B*T, D, vocab]"""
    codes = codes.view(codes.shape[0], -1, codes.shape[-1])                                   # :374
    e = F.embedding(codes, sd["tok_emb_code.weight"])                                         # :375
    xc = F.embedding(conds, sd["tok_emb_cond.weight"]) + sd["pos_emb_cond"]                   # :376, :382
    cs = e.cumsum(-1)                                           # :378 -- over the CHANNEL axis, not over depth
    xi = cs[..., -1, :] + sd["pos_emb_code"]                    # :379, :381 -- only the last depth's code enters
    Tc = conds.shape[1]
    h = torch.cat([xc, xi], dim=1)                                                            # :384
    for i in range(n_layers_of(sd, "spatial_transformer")):
        h = block(sd, f"spatial_transformer.{i}.", h, spatial_heads, Tc)                     # :385
    h = _ln(h, sd["ln_spatial.weight"], sd["ln_spatial.bias"])[:, Tc - 1:-1]                  # :385-386
    v = cs[..., :-1, :] + sd["pos_emb_depth"]                                                 # :388
    v = torch.cat([h.unsqueeze(2), v], dim=2)                                                 # :389
    v = v.reshape(-1, *v.shape[2:])                                                           # :391
    for i in range(n_layers_of(sd, "depth_transformer")):
        v = block(sd, f"depth_transformer.{i}.", v, depth_heads, 0)                          # :392
    return F.linear(_ln(v, sd["ln_depth.weight"], sd["ln_depth.bias"]), sd["head.weight"])    # :393


def rq_loss(sd, codes, conds, spatial_heads, depth_heads):
    """CondTransformer.shared_step, stage2/transformer.py:117-118"""
    logits = rq_forward(sd, codes, conds, spatial_heads, depth_heads)
    return F.cross_entropy(logits.reshape(-1, logits.shape[-1]), codes.reshape(-1)), logits


def _cached_block(sd, p, x, n_heads, past):
    """Block.sample with layer_past (layers.py:138-143, :57-81 with use_cache): one token, the shifted input all zero (:58 on
    T == 1), its key / value appended to the cache, attention over the cache unmasked"""
    B, _, C = x.shape
    hs = C // n_heads
    h = time_mix(_ln(x, sd[p + "ln1.weight"], sd[p + "ln1.bias"]), sd[p + "attn.time_mix"])

    def lin(name, v_):
        return F.linear(v_, sd[p + "attn." + name + ".weight"], sd.get(p + "attn." + name + ".bias"))
    k = lin("key", h).view(B, 1, n_heads, hs).transpose(1, 2)
    q = lin("query", h).view(B, 1, n_heads, hs).transpose(1, 2)
    v = lin("value", h).view(B, 1, n_heads, hs).transpose(1, 2)
    past[0] = k if past[0] is None else torch.cat([past[0], k], dim=-2)
    past[1] = v if past[1] is None else torch.cat([past[1], v], dim=-2)
    att = F.softmax(q @ (past[0].transpose(-2, -1) * (1.0 / math.sqrt(hs))), dim=-1)
    y = (att @ past[1]).transpose(1, 2).reshape(B, 1, C)
    x = x + lin("proj", y)
    return x + ffn(sd, p + "mlp.", _ln(x, sd[p + "ln2.weight"], sd[p + "ln2.bias"]))


def rq_sample_logits(sd, conds, codes, spatial_heads, depth_heads):
    """The logits RQTransformer.sample (layers.py:397-547) computes step by step when it draws exactly `codes` [B, T, D]:
    [B*T, D, vocab].  Follows sample_spatial_step / sample_depth_step literally, with their quirks: a spatial step embeds the
    previous position's codes as a sum over depth (:502), a depth step d > 0 the sum of this position's codes so far
    (:535); depth step 0 applies ln_depth twice (:531, :542); one-token steps mix with an all-zero shift and attend to
    the cache unmasked."""
    B, T, D = codes.shape
    Ls, Ld = n_layers_of(sd, "spatial_transformer"), n_layers_of(sd, "depth_transformer")
    Tc = conds.shape[1]
    W = sd["tok_emb_code.weight"]
    ln_d = lambda t: _ln(t, sd["ln_depth.weight"], sd["ln_depth.bias"])          # noqa: E731
    x = F.embedding(conds, sd["tok_emb_cond.weight"]) + sd["pos_emb_cond"]       # :491-492
    spast = []
    for i in range(Ls):
        p = f"spatial_transformer.{i}."
        a, k, v = attention(sd, p + "attn.", _ln(x, sd[p + "ln1.weight"], sd[p + "ln1.bias"]), spatial_heads, Tc)
        spast.append([k, v])
        x = x + a
        x = x + ffn(sd, p + "mlp.", _ln(x, sd[p + "ln2.weight"], sd[p + "ln2.bias"]))
    hidden = _ln(x, sd["ln_spatial.weight"], sd["ln_spatial.bias"])[:, Tc - 1:Tc]            # :497-498
    out = []
    for t in range(T):
        if t > 0:
            x = F.embedding(codes[:, t - 1], W).sum(1, keepdim=True) + sd["pos_emb_code"][:, t - 1:t]   # :501-502
            for i in range(Ls):
                x = _cached_block(sd, f"spatial_transformer.{i}.", x, spatial_heads, spast[i])
            hidden = _ln(x, sd["ln_spatial.weight"], sd["ln_spatial.bias"])[:, -1:]                  # :509-510
        dpast = [[None, None] for _ in range(Ld)]
        for d in range(D):
            if d == 0:
                x = hidden                                                                            # :526
            else:
                x = F.embedding(codes[:, t, :d], W).sum(1, keepdim=True) + sd["pos_emb_depth"][:, d - 1:d]   # :534-535
            for i in range(Ld):
                x = _cached_block(sd, f"depth_transformer.{i}.", x, depth_heads, dpast[i])
            y = ln_d(ln_d(x)) if d == 0 else ln_d(x)                                                  # :531, :542
            out.append(F.linear(y[:, -1], sd["head.weight"]))                                         # :543-545
    return torch.stack(out, 1).view(B * T, D, -1)
