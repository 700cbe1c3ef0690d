"""Drop-in ``GPT`` (and its ``Block`` / ``MultiHeadSelfAttention`` / ``FFN``) for the reference's
``enhancing/modules/stage2/layers.py`` -- SURVEY.md section 8f-3, BASELINE config 5.

Same constructor keywords (``stage2/transformer.py:41`` instantiates the YAML's ``transformer`` target), same
``forward(codes, conds) -> logits`` / ``sample`` / ``sample_step`` signatures, same ``state_dict`` keys and
shapes, same module classes (``configure_optimizers`` sorts parameters by ``isinstance(m, nn.Linear)`` etc.,
``stage2/transformer.py:141-160``), but every FLOP runs in libb200vq.so: the seven Linear layers of a block and
the vocabulary head on the tensor-core GEMMs, the masked attention core on the tf32 / 3xTF32 kernels with the
causal + visible-prefix mask folded in, time-shift mixing, squared ReLU, embeddings and the logits window as
HBM streams (csrc/stage2.cu).

Data path (``etb.set_precision``): "fp16" (default) -> the Linear layers on f16 GEMMs (fp16 operands, fp32 accumulate and
output, per-call power-of-two gradient scaling chosen on the device), attention core on tf32; "tf32" -> everything
tf32; "parity" -> 3xTF32 GEMMs and attention (fp32-grade).  Limits of the kernels underneath, raised at construction:
head size ``embed_dim // n_heads`` must be 32, 64, 96 or 128, ``embed_dim`` <= 2048 and a multiple of 64, ``vocab_img_size`` % 64 == 0
(the YAML's 6144 / 16 = 384-wide heads -- a 10.9 B-parameter model that cannot train under replicated fp32 DDP anyway, SURVEY.md
section 8f-3 -- are not covered).  Heads of 96 and 128 run on wide-head kernels that keep their resident operands in shared
memory (DESIGN.md section 4.2); 32 and 64 on the register-resident ones.

``RQTransformer`` (reference :306-547, the prior over residual codes [B, T, D]) reuses these blocks: its spatial transformer is
``GPT``'s, its depth transformer runs causal attention over B*T sequences of D <= 16 tokens on the short-sequence kernel of
csrc/rq_stage2.cu (fp32 FMA on every data path), and its channel-cumsum code embeddings are HBM streams there too.

There is no CPU path: CPU tensors raise (use the reference classes on CPU)."""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch
import torch.nn as nn
from torch.nn import functional as F

from . import functional as Fn
from . import ops
from .layers import _flat2d

Tensor = torch.Tensor
_fwd, _bwd = Fn._fwd, Fn._bwd


def _mode() -> str:
    """data path of the attention core and of everything that is not a Linear: "parity" (3xTF32) or "tf32" """
    return "parity" if Fn.get_precision() == "parity" else "tf32"


def _linear(x: Tensor, w: Tensor, b: Optional[Tensor], res: Optional[Tensor] = None) -> Tensor:
    """x W^T + b (+ res) on the data path `etb.set_precision` selects: fp16 tensor-core operands (default), tf32, or 3xTF32"""
    if Fn.get_precision() == "fp16":
        return LinearF16Fn.apply(x, w, b, res)
    if res is None:
        return Fn.LinearFn.apply(x, w, b, 0, False)
    return LinearResFn.apply(x, w, b, res)


class TokenEmbedFn(torch.autograd.Function):
    """cat(tok_emb_cond(conds) + pos_emb_cond, tok_emb_code(codes) + pos_emb_code) (reference stage2/layers.py:199-206)"""

    @staticmethod
    def forward(ctx, conds, codes, Wc, pos_c, Wi, pos_i):
        x = ops.token_embed_fwd(conds, codes, Wc, pos_c, Wi, pos_i)
        ctx.save_for_backward(conds, codes)
        ctx.vocab = (Wc.shape[0], Wi.shape[0], pos_c.shape, pos_i.shape)
        return x

    @staticmethod
    def backward(ctx, g):
        conds, codes = ctx.saved_tensors
        Vc, Vi, shape_c, shape_i = ctx.vocab
        bwd = ops.token_embed_bwd_deterministic if Fn.deterministic() else ops.token_embed_bwd
        gWc, gpc, gWi, gpi = bwd(conds, codes, g.contiguous(), Vc, Vi)
        return None, None, gWc, gpc.view(shape_c), gWi, gpi.view(shape_i)


class TimeMixFn(torch.autograd.Function):
    """x * time_mix + time_shift(x) * (1 - time_mix) (reference stage2/layers.py:50-58)"""

    @staticmethod
    @_fwd
    def forward(ctx, x, w, T):
        ctx.save_for_backward(x, w)
        ctx.T = T
        return ops.time_mix_fwd(x, w.view(-1), T)

    @staticmethod
    @_bwd
    def backward(ctx, g):
        x, w = ctx.saved_tensors
        gx, gw = ops.time_mix_bwd(g.contiguous(), x, w.view(-1), ctx.T)
        return gx, gw.view_as(w), None


class SqReluFn(torch.autograd.Function):
    """torch.square(torch.relu(x)) (reference stage2/layers.py:108)"""

    @staticmethod
    @_fwd
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return ops.sqrelu(x)

    @staticmethod
    @_bwd
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        return ops.sqrelu(x, g.contiguous())


class LinearResFn(torch.autograd.Function):
    """res + x W^T + b: a block's output projections with the skip connection added in the GEMM epilogue
    (reference stage2/layers.py:91,110 with :131-132)"""

    @staticmethod
    @_fwd
    def forward(ctx, x, w, b, res):
        M, K = x.shape
        N = w.shape[0]
        mode = _mode()
        xr = x if mode == "parity" else ops.round_tf32(x)
        y = Fn._mm(xr, Fn._W(w, mode), M, N, K, mode, bias=b, res=res)
        ctx.save_for_backward(xr, w)
        ctx.cfg = (b is not None, mode)
        return y

    @staticmethod
    @_bwd
    def backward(ctx, g):
        xr, w = ctx.saved_tensors
        has_bias, mode = ctx.cfg
        M, K = xr.shape
        N = w.shape[0]
        g = g.contiguous()
        gr = g if mode == "parity" else ops.round_tf32(g)
        need_x, need_w, need_b, need_res = ctx.needs_input_grad[:4]
        db = ops.colsum(gr) if (has_bias and need_b) else None
        dw = Fn._wgrad(gr, xr, N, K, mode) if need_w else None
        dx = Fn._mm(gr, Fn._W(w, mode, True), M, K, N, mode, b_major=1) if need_x else None
        return dx, dw, db, (g if need_res else None)


class LinearF16Fn(torch.autograd.Function):
    """x W^T + b (+ res) with fp16 tensor-core operands and fp32 accumulation / output (fp16: tf32's 11-bit significand
    at twice the tensor rate and half the operand bytes -- DESIGN.md section 2).  Self-contained gradient scaling: backward
    picks the power of two S that puts max|g| at 2^6 on the device (`ops.grad_scale`, no host sync), feeds fp16(g S) to the
    dgrad / wgrad GEMMs and multiplies their fp32 results by 1/S in the epilogue (exact)."""

    @staticmethod
    @_fwd
    def forward(ctx, x, w, b, res):
        M, K = x.shape
        N = w.shape[0]
        x16 = ops.to_half(x)
        y = ops.gemm(x16, Fn.weight_shadow(w, "f16"), M, N, K, bias=b, res=res, cta_group=Fn.GEMM_CTA_GROUP)
        ctx.save_for_backward(x16, w)
        ctx.has_bias = b is not None
        return y

    @staticmethod
    @_bwd
    def backward(ctx, g):
        x16, w = ctx.saved_tensors
        M, K = x16.shape
        N = w.shape[0]
        g = g.contiguous()
        need_x, need_w, need_b, need_res = ctx.needs_input_grad[:4]
        sc = ops.grad_scale(g)
        gh = ops.to_half(g, sc[0:1])
        db = ops.colsum(g) if (ctx.has_bias and need_b) else None
        dw = Fn._wgrad(gh, x16, N, K, inv_scale=sc[1:2]) if need_w else None
        dx = ops.gemm(gh, Fn.weight_shadow(w, "f16", True), M, K, N, b_major=1, alpha=sc[1:2], cta_group=Fn.GEMM_CTA_GROUP) if need_x else None
        return dx, dw, db, (g if need_res else None)


class CausalAttentionFn(torch.autograd.Function):
    """softmax(mask(q k^T / sqrt(hs))) v on the packed qkv matrix (reference stage2/layers.py:76-89): the mask is
    tril with the cond_len x cond_len prefix block fully visible (:43-48)."""

    @staticmethod
    @_fwd
    def forward(ctx, qkv, B, T, heads, hs, cond_len):
        scale = 1.0 / math.sqrt(hs)
        exact = _mode() == "parity"
        qr = qkv if exact else ops.round_tf32(qkv)
        o, lse = ops.attention_causal_fwd(qr, B, T, heads, hs, scale, cond_len, exact)
        ctx.save_for_backward(qr, o, lse)
        ctx.dims = (B, T, heads, hs, cond_len, exact, scale)
        return o

    @staticmethod
    @_bwd
    def backward(ctx, g):
        qr, o, lse = ctx.saved_tensors
        B, T, heads, hs, cond_len, exact, scale = ctx.dims
        g = g.contiguous()
        if not exact:
            g = ops.round_tf32(g)
        dqkv = ops.attention_causal_bwd(qr, o, lse, g, B, T, heads, hs, scale, cond_len, exact)
        return dqkv, None, None, None, None, None


class RowWindowFn(torch.autograd.Function):
    """x[:, off:off+n] of a [B*T, C] matrix as a contiguous [B*n, C] one (reference stage2/layers.py:210)"""

    @staticmethod
    @_fwd
    def forward(ctx, x, B, T, off, n):
        ctx.geom = (B, T, off, n)
        return ops.copy_rows(x, B, T, n, off, 0, n)

    @staticmethod
    @_bwd
    def backward(ctx, g):
        B, T, off, n = ctx.geom
        return ops.copy_rows(g.contiguous(), B, n, T, 0, off, n), None, None, None, None


class ShortAttentionFn(torch.autograd.Function):
    """the masked attention core over nseq independent sequences of D <= 16 tokens (the depth transformer's blocks,
    reference stage2/layers.py:346-352 with ctx_len = D, cond_len = 0): one warp per (sequence, head), fp32 FMA"""

    @staticmethod
    @_fwd
    def forward(ctx, qkv, nseq, D, heads, hs, cond_len):
        scale = 1.0 / math.sqrt(hs)
        ctx.save_for_backward(qkv)
        ctx.dims = (nseq, D, heads, hs, cond_len, scale)
        return ops.short_attention_fwd(qkv, nseq, D, heads, hs, scale, cond_len)

    @staticmethod
    @_bwd
    def backward(ctx, g):
        (qkv,) = ctx.saved_tensors
        nseq, D, heads, hs, cond_len, scale = ctx.dims
        return ops.short_attention_bwd(qkv, g.contiguous(), nseq, D, heads, hs, scale, cond_len), None, None, None, None, None


class RQEmbedFn(torch.autograd.Function):
    """the spatial input of RQTransformer.forward (reference stage2/layers.py:374-384): cat(tok_emb_cond(conds) + pos_emb_cond,
    tok_emb_code(codes).cumsum(-1)[..., -1, :] + pos_emb_code) -- the cumsum runs over the channels, so only the last depth's
    code enters"""

    @staticmethod
    def forward(ctx, conds, codes, Wc, pos_c, Wi, pos_i):
        ctx.save_for_backward(conds, codes)
        ctx.vocab = (Wc.shape[0], Wi.shape[0], pos_c.shape, pos_i.shape)
        return ops.rq_embed_fwd(conds, codes, Wc, pos_c, Wi, pos_i)

    @staticmethod
    def backward(ctx, g):
        conds, codes = ctx.saved_tensors
        Vc, Vi, shape_c, shape_i = ctx.vocab
        gWc, gpc, gWi, gpi = ops.rq_embed_bwd(conds, codes, g.contiguous(), Vc, Vi, deterministic=Fn.deterministic())
        return None, None, gWc, gpc.view(shape_c), gWi, gpi.view(shape_i)


class RQDepthInputFn(torch.autograd.Function):
    """the depth input of RQTransformer.forward (reference stage2/layers.py:388-391): per code position, row 0 is the spatial
    hidden state h, row d >= 1 is tok_emb_code(codes[..., d-1]).cumsum(-1) + pos_emb_depth[d-1]"""

    @staticmethod
    def forward(ctx, h, codes, Wi, pos_d):
        ctx.save_for_backward(codes)
        ctx.meta = (Wi.shape[0], pos_d.shape)
        return ops.rq_depth_input_fwd(h, codes, Wi, pos_d)

    @staticmethod
    def backward(ctx, g):
        (codes,) = ctx.saved_tensors
        Vi, shape_d = ctx.meta
        gh, gWi, gpd = ops.rq_depth_input_bwd(codes, g.contiguous(), Vi, deterministic=Fn.deterministic())
        return gh, None, gWi, gpd.view(shape_d)


HEAD_SIZES = (32, 64, 96, 128)    # head sizes the attention, KV-cache and depth kernels take


def _check_kernel_limits(embed_dim: int, n_heads: int) -> None:
    assert embed_dim % n_heads == 0
    hs = embed_dim // n_heads
    if hs not in HEAD_SIZES:
        raise NotImplementedError(f"b200vq stage 2: head size embed_dim // n_heads must be 32, 64, 96 or 128 (got {hs}); "
                                  "use the reference modules for this geometry")
    if embed_dim > 2048 or embed_dim % 64:
        raise NotImplementedError(f"b200vq stage 2: embed_dim must be a multiple of 64 and <= 2048 (got {embed_dim})")


class MultiHeadSelfAttention(nn.Module):
    """reference stage2/layers.py:23-96; `key` / `query` / `value` / `proj` / `time_mix` hold the parameters"""

    def __init__(self, ctx_len: int, cond_len: int, embed_dim: int, n_heads: int, attn_bias: bool, use_mask: bool = True) -> None:
        super().__init__()
        _check_kernel_limits(embed_dim, n_heads)
        self.key = nn.Linear(embed_dim, embed_dim, bias=attn_bias)
        self.query = nn.Linear(embed_dim, embed_dim, bias=attn_bias)
        self.value = nn.Linear(embed_dim, embed_dim, bias=attn_bias)
        self.proj = nn.Linear(embed_dim, embed_dim, attn_bias)
        self.n_heads, self.ctx_len, self.cond_len, self.use_mask = n_heads, ctx_len, cond_len, use_mask
        # set by RQTransformer on its depth blocks: B*T sequences of ctx_len <= 16 tokens go to the short-sequence kernel
        self.short_seq = False
        if use_mask:       # never read by the kernels (the mask is two integers there); kept for module-tree parity
            mask = torch.tril(torch.ones(ctx_len, ctx_len)).view(1, ctx_len, ctx_len)
            mask[:, :cond_len, :cond_len] = 1
            self.register_buffer("mask", mask, persistent=False)
        self.time_shift = nn.ZeroPad2d((0, 0, 1, -1))
        ramp = torch.arange(embed_dim, dtype=torch.float32) / (embed_dim - 1)
        self.time_mix = nn.Parameter(ramp.view(1, 1, embed_dim))

    def packed_qkv(self) -> Tuple[Tensor, Optional[Tensor]]:
        """[3C, C] weight (+ [3C] bias) in the q | k | v order the attention kernels read"""
        w = torch.cat([self.query.weight, self.key.weight, self.value.weight], dim=0)
        b = None if self.query.bias is None else torch.cat([self.query.bias, self.key.bias, self.value.bias], dim=0)
        return w, b

    def core(self, flat: Tensor, B: int, T: int, res: Optional[Tensor] = None) -> Tensor:
        """flat [B*T, C] (the LayerNorm output) -> proj(attention(time_mix(flat))) (+ res)"""
        C = flat.shape[-1]
        mixed = TimeMixFn.apply(flat, self.time_mix, T)
        w, b = self.packed_qkv()
        qkv = _linear(mixed, w, b)
        cond = min(self.cond_len, T) if self.use_mask else T      # no mask == every key visible == a prefix of T tokens
        if self.short_seq:
            o = ShortAttentionFn.apply(qkv, B, T, self.n_heads, C // self.n_heads, cond)
        else:
            o = CausalAttentionFn.apply(qkv, B, T, self.n_heads, C // self.n_heads, cond)
        return _linear(o, self.proj.weight, self.proj.bias, res)

    def forward(self, x: Tensor, use_cache: bool = False, layer_past=None):
        if use_cache or layer_past is not None:
            raise NotImplementedError("b200vq stage 2: the KV cache lives in GPT.sample (one preallocated buffer per layer), "
                                      "not in per-call tensors; call GPT.sample / GPT.sample_step")
        B, T, C = x.shape
        return self.core(_flat2d(x), B, T).view(B, T, C)


class FFN(nn.Module):
    """reference stage2/layers.py:98-111: Linear -> square(relu) -> Linear"""

    def __init__(self, embed_dim: int, mlp_bias: bool) -> None:
        super().__init__()
        self.p0 = nn.Linear(embed_dim, 4 * embed_dim, bias=mlp_bias)
        self.p1 = nn.Linear(4 * embed_dim, embed_dim, bias=mlp_bias)

    def core(self, flat: Tensor, res: Optional[Tensor] = None) -> Tensor:
        # the squared ReLU stays a stream kernel of its own: folded into the GEMM epilogue (measured, same box) it cost the
        # stage-1 GEMMs 2 % through the larger epilogue code, for a gain that only stage 2 sees
        hidden = SqReluFn.apply(_linear(flat, self.p0.weight, self.p0.bias))
        return _linear(hidden, self.p1.weight, self.p1.bias, res)

    def forward(self, x: Tensor) -> Tensor:
        return self.core(_flat2d(x)).view(*x.shape[:-1], -1)


class Block(nn.Module):
    """reference stage2/layers.py:113-143"""

    def __init__(self, ctx_len: int, cond_len: int, embed_dim: int, n_heads: int, mlp_bias: bool, attn_bias: bool) -> None:
        super().__init__()
        self.ln1 = nn.LayerNorm(embed_dim)
        self.ln2 = nn.LayerNorm(embed_dim)
        self.attn = MultiHeadSelfAttention(ctx_len=ctx_len, cond_len=cond_len, embed_dim=embed_dim, n_heads=n_heads,
                                           attn_bias=attn_bias, use_mask=True)
        self.mlp = FFN(embed_dim=embed_dim, mlp_bias=mlp_bias)

    def run(self, flat: Tensor, B: int, T: int) -> Tensor:
        """flat [B*T, C] -> flat [B*T, C]; both skip connections ride the output GEMMs' epilogues"""
        h = Fn.LayerNormFn.apply(flat, self.ln1.weight, self.ln1.bias, False)
        flat = self.attn.core(h, B, T, res=flat)
        h = Fn.LayerNormFn.apply(flat, self.ln2.weight, self.ln2.bias, False)
        return self.mlp.core(h, res=flat)

    def forward(self, x: Tensor) -> Tensor:
        B, T, C = x.shape
        return self.run(_flat2d(x), B, T).view(B, T, C)

    def sample(self, x, layer_past=None):
        raise NotImplementedError("b200vq stage 2: use GPT.sample / GPT.sample_step (the KV cache is owned by GPT)")


def _cached_prefix(blocks, x: Tensor, B: int, T: int, ctx: int, heads: int, hs: int):
    """the first sampling step of a block stack (reference stage2/layers.py:139-143 with layer_past None) over x [B*T, C]:
    T tokens that see each other fully (the condition prefix, :83-85 with T == cond_len; or one token).  Allocates each
    layer's key / value cache [B, ctx, C] and fills its first T rows.  -> (x, past)"""
    C = x.shape[-1]
    past = {"k": [], "v": [], "len": T}
    for block in blocks:
        att = block.attn
        h = Fn.LayerNormFn.apply(x, block.ln1.weight, block.ln1.bias, False)
        mixed = ops.time_mix_fwd(h, att.time_mix.view(-1), T)
        w, b = att.packed_qkv()
        qkv = _linear(mixed, w, b)
        ck = torch.zeros(B, ctx, C, device=x.device)
        cv = torch.zeros(B, ctx, C, device=x.device)
        q3 = qkv.view(B, T, 3, C)
        ck[:, :T] = q3[:, :, 1]
        cv[:, :T] = q3[:, :, 2]
        past["k"].append(ck)
        past["v"].append(cv)
        o = CausalAttentionFn.apply(qkv, B, T, heads, hs, T)
        x = _linear(o, att.proj.weight, att.proj.bias, x)
        x = block.mlp.core(Fn.LayerNormFn.apply(x, block.ln2.weight, block.ln2.bias, False), res=x)
    return x, past


def _cached_step(blocks, x: Tensor, past: dict, heads: int, hs: int) -> Tensor:
    """one later sampling step of a block stack over x [B, C] (reference stage2/layers.py:139-143 with layer_past): the key /
    value rows go to cache row past["len"], the query attends to rows 0 .. past["len"] unmasked (:76-81)"""
    pos = past["len"]
    scale = 1.0 / math.sqrt(hs)
    for li, block in enumerate(blocks):
        att = block.attn
        h = Fn.LayerNormFn.apply(x, block.ln1.weight, block.ln1.bias, False)
        mixed = ops.time_mix_fwd(h, att.time_mix.view(-1), 1)
        w, b = att.packed_qkv()
        qkv = _linear(mixed, w, b)
        o = ops.decode_attention(qkv, past["k"][li], past["v"][li], heads, hs, pos, scale)
        x = _linear(o, att.proj.weight, att.proj.bias, x)
        x = block.mlp.core(Fn.LayerNormFn.apply(x, block.ln2.weight, block.ln2.bias, False), res=x)
    past["len"] = pos + 1
    return x


def _filter_and_draw(logits_: Tensor, top_k, top_p) -> Tensor:
    """the top-k / nucleus filtering and multinomial draw of the reference's samplers (stage2/layers.py:242-260, :448-466),
    call for call, so that the same torch RNG stream draws the same codes"""
    if top_k is not None:
        v, ix = torch.topk(logits_, top_k)
        logits_[logits_ < v[:, [-1]]] = -float('Inf')
    probs = F.softmax(logits_, dim=-1)
    if top_p is not None:
        sorted_probs, sorted_indices = torch.sort(probs, dim=-1, descending=True)
        cum_probs = torch.cumsum(sorted_probs, dim=-1)
        remove = cum_probs >= top_p
        remove[..., 1:] = remove[..., :-1].clone()
        remove[..., 0] = 0
        probs = probs.masked_fill(remove.scatter(-1, sorted_indices, remove), 0.0)
        probs = probs / torch.sum(probs, dim=-1, keepdim=True)
    return torch.multinomial(probs, num_samples=1).clone().detach()


class GPT(nn.Module):
    """reference stage2/layers.py:146-303"""

    def __init__(self, vocab_cond_size: int, vocab_img_size: int, embed_dim: int, cond_num_tokens: int, img_num_tokens: int,
                 n_heads: int, n_layers: int, mlp_bias: bool = True, attn_bias: bool = True) -> None:
        super().__init__()
        if vocab_img_size % 64:
            # the head's weight gradient reads d(logits) as an MN-major tensor-core operand: whole 64-column (fp16) atoms
            raise NotImplementedError(f"b200vq stage 2: vocab_img_size must be a multiple of 64 (got {vocab_img_size})")
        self.img_num_tokens = img_num_tokens
        self.vocab_cond_size = vocab_cond_size
        self.tok_emb_cond = nn.Embedding(vocab_cond_size, embed_dim)
        self.pos_emb_cond = nn.Parameter(torch.zeros(1, cond_num_tokens, embed_dim))
        self.tok_emb_code = nn.Embedding(vocab_img_size, embed_dim)
        self.pos_emb_code = nn.Parameter(torch.zeros(1, img_num_tokens, embed_dim))
        ctx = cond_num_tokens + img_num_tokens
        self.blocks = nn.Sequential(*[Block(ctx_len=ctx, cond_len=cond_num_tokens, embed_dim=embed_dim, n_heads=n_heads,
                                            mlp_bias=mlp_bias, attn_bias=attn_bias) for _ in range(n_layers)])
        self.layer_norm = nn.LayerNorm(embed_dim)
        self.head = nn.Linear(embed_dim, vocab_img_size, bias=False)
        self.apply(self._init_weights)

    def _init_weights(self, module: nn.Module) -> None:
        """reference stage2/layers.py:184-192: N(0, 0.02) matrices / embeddings, zero biases, unit LayerNorm"""
        if isinstance(module, (nn.Linear, nn.Embedding)):
            module.weight.data.normal_(mean=0.0, std=0.02)
            if isinstance(module, nn.Linear) and module.bias is not None:
                module.bias.data.zero_()
        elif isinstance(module, nn.LayerNorm):
            module.bias.data.zero_()
            module.weight.data.fill_(1.0)

    def forward(self, codes: torch.LongTensor, conds: torch.LongTensor) -> torch.FloatTensor:
        codes = codes.view(codes.shape[0], -1).contiguous()
        conds = conds.contiguous()
        B, Tc = conds.shape
        Ti = codes.shape[1]
        assert Ti == self.pos_emb_code.shape[1] and Tc == self.pos_emb_cond.shape[1], \
            "codes / conds must have img_num_tokens / cond_num_tokens entries (the positional tables are added whole)"
        T = Tc + Ti
        x = TokenEmbedFn.apply(conds, codes, self.tok_emb_cond.weight, self.pos_emb_cond, self.tok_emb_code.weight, self.pos_emb_code)
        for block in self.blocks:
            x = block.run(x, B, T)
        x = Fn.LayerNormFn.apply(x, self.layer_norm.weight, self.layer_norm.bias, False)
        x = RowWindowFn.apply(x, B, T, Tc - 1, Ti)                    # positions cond-1 .. T-2 predict the Ti codes
        logits = _linear(x, self.head.weight, None)
        return logits.view(B, Ti, -1)

    # ------------------------------------------------------------------------------------------ sampling
    @torch.no_grad()
    def sample(self, conds: torch.LongTensor, top_k: Optional[float] = None, top_p: Optional[float] = None,
               softmax_temperature: float = 1.0, use_fp16: bool = True) -> Tuple[torch.FloatTensor, torch.LongTensor]:
        """reference stage2/layers.py:213-262.  The filtering / multinomial draw are the reference's own torch calls on
        the [B, vocab] logits (so the same torch RNG stream yields the same codes); the transformer steps run in
        libb200vq.so with one preallocated KV cache per layer instead of per-step `torch.cat`s.  `use_fp16` (an autocast
        switch in the reference) is accepted and ignored: the kernels' precision is `etb.set_precision`."""
        past = codes = logits = None
        for i in range(self.img_num_tokens):
            if codes is None:
                codes_, pos_code = None, None
            else:
                codes_ = codes.clone().detach()[:, -1:]
                pos_code = self.pos_emb_code[:, i - 1:i, :]
            logits_, past = self.sample_step(codes_, conds, pos_code, use_fp16, past)
            logits_ = logits_.to(dtype=torch.float32) / softmax_temperature
            idx = _filter_and_draw(logits_, top_k, top_p)
            codes = idx if codes is None else torch.cat([codes, idx], axis=1)
            logits = logits_ if logits is None else torch.cat([logits, logits_], axis=1)
        del past
        return logits, codes

    @torch.no_grad()
    def sample_step(self, codes, conds, pos_code, use_fp16: bool = True, past=None):
        """reference stage2/layers.py:264-303.  `past` is this implementation's cache object: a dict with per-layer key / value
        buffers [B, ctx_len, C] and the number of rows filled (None on the first step, as in the reference)."""
        C = self.head.weight.shape[1]
        heads = self.blocks[0].attn.n_heads if len(self.blocks) else 1
        hs = C // heads
        if codes is None:
            assert past is None
            conds = conds.contiguous()
            B, Tc = conds.shape
            ctx = Tc + self.img_num_tokens
            dev = self.head.weight.device
            empty = torch.empty(B, 0, dtype=torch.int64, device=dev)
            x = ops.token_embed_fwd(conds, empty, self.tok_emb_cond.weight, self.pos_emb_cond.view(Tc, C),
                                    self.tok_emb_code.weight, self.pos_emb_code.view(-1, C))
            x, past = _cached_prefix(self.blocks, x, B, Tc, ctx, heads, hs)
            x = Fn.LayerNormFn.apply(x, self.layer_norm.weight, self.layer_norm.bias, False)
            x = ops.copy_rows(x, B, Tc, 1, Tc - 1, 0, 1)
        else:
            assert past is not None
            B = codes.shape[0]
            # a one-token sequence: time_shift(x) is all zeros (reference :58 on T == 1), so the mix is x * time_mix + 0
            x = ops.token_embed_fwd(torch.empty(B, 0, dtype=torch.int64, device=codes.device), codes.contiguous().view(B, 1),
                                    self.tok_emb_cond.weight, self.pos_emb_cond.view(-1, C), self.tok_emb_code.weight,
                                    pos_code.contiguous().view(1, C))
            x = _cached_step(self.blocks, x, past, heads, hs)
            x = Fn.LayerNormFn.apply(x, self.layer_norm.weight, self.layer_norm.bias, False)
        logits = _linear(x, self.head.weight, None)
        return logits, past


class RQTransformer(nn.Module):
    """reference stage2/layers.py:306-547: a spatial transformer over the code positions and a depth transformer over the D
    residual codes of each position.  Reproduces what the reference computes, quirks included: the code embeddings are
    prefix sums over the channel axis (`cumsum(-1)`, :378), the sampler embeds codes as sums over depth (:502, :535) and
    applies `ln_depth` twice on depth step 0 (:531, :542).  Limits of the kernels underneath, raised at construction: head
    sizes 32 / 64 / 96 / 128 (spatial and depth, chosen independently), `embed_dim` <= 2048 and a multiple of 64,
    `vocab_img_size` % 64 == 0, 2 <= `depth_num_tokens` <= 16."""

    def __init__(self, vocab_cond_size: int, vocab_img_size: int, embed_dim: int, cond_num_tokens: int, img_num_tokens: int,
                 depth_num_tokens: int, spatial_n_heads: int, depth_n_heads: int, spatial_n_layers: int, depth_n_layers: int,
                 mlp_bias: bool = True, attn_bias: bool = True) -> None:
        super().__init__()
        if vocab_img_size % 64:
            raise NotImplementedError(f"b200vq stage 2: vocab_img_size must be a multiple of 64 (got {vocab_img_size})")
        if not 2 <= depth_num_tokens <= 16:
            # the short-sequence attention kernel holds a whole depth sequence per warp
            raise NotImplementedError(f"b200vq stage 2: depth_num_tokens must be in 2..16 (got {depth_num_tokens})")
        _check_kernel_limits(embed_dim, spatial_n_heads)
        _check_kernel_limits(embed_dim, depth_n_heads)
        self.img_num_tokens = img_num_tokens
        self.depth_num_tokens = depth_num_tokens
        self.vocab_img_size = vocab_img_size
        self.tok_emb_cond = nn.Embedding(vocab_cond_size, embed_dim)
        self.pos_emb_cond = nn.Parameter(torch.rand(1, cond_num_tokens, embed_dim))
        self.tok_emb_code = nn.Embedding(vocab_img_size, embed_dim)
        self.pos_emb_code = nn.Parameter(torch.rand(1, img_num_tokens, embed_dim))
        self.pos_emb_depth = nn.Parameter(torch.rand(1, depth_num_tokens - 1, embed_dim))
        self.spatial_transformer = nn.Sequential(*[Block(ctx_len=cond_num_tokens + img_num_tokens, cond_len=cond_num_tokens,
                                                         embed_dim=embed_dim, n_heads=spatial_n_heads, mlp_bias=mlp_bias,
                                                         attn_bias=attn_bias) for _ in range(spatial_n_layers)])
        self.depth_transformer = nn.Sequential(*[Block(ctx_len=depth_num_tokens, cond_len=0, embed_dim=embed_dim,
                                                       n_heads=depth_n_heads, mlp_bias=mlp_bias, attn_bias=attn_bias)
                                                 for _ in range(depth_n_layers)])
        for block in self.depth_transformer:
            block.attn.short_seq = True
        self.ln_spatial = nn.LayerNorm(embed_dim)
        self.ln_depth = nn.LayerNorm(embed_dim)
        self.head = nn.Linear(embed_dim, vocab_img_size, bias=False)
        self.apply(self._init_weights)

    _init_weights = GPT._init_weights

    def forward(self, codes: torch.LongTensor, conds: torch.LongTensor) -> torch.FloatTensor:
        """reference stage2/layers.py:370-395: codes [B, T, D], conds [B, Tc] -> logits [B*T, D, vocab_img_size]"""
        D = codes.shape[-1]
        codes = codes.reshape(codes.shape[0], -1, D).contiguous()
        conds = conds.contiguous()
        B, Tc = conds.shape
        T = codes.shape[1]
        assert D == self.depth_num_tokens and T == self.pos_emb_code.shape[1] and Tc == self.pos_emb_cond.shape[1], \
            "codes / conds must be [B, img_num_tokens, depth_num_tokens] / [B, cond_num_tokens] (the positional tables are added whole)"
        x = RQEmbedFn.apply(conds, codes, self.tok_emb_cond.weight, self.pos_emb_cond, self.tok_emb_code.weight, self.pos_emb_code)
        for block in self.spatial_transformer:
            x = block.run(x, B, Tc + T)
        x = Fn.LayerNormFn.apply(x, self.ln_spatial.weight, self.ln_spatial.bias, False)
        h = RowWindowFn.apply(x, B, Tc + T, Tc - 1, T)                 # positions cond-1 .. Tc+T-2 (:386)
        v = RQDepthInputFn.apply(h, codes, self.tok_emb_code.weight, self.pos_emb_depth)
        for block in self.depth_transformer:
            v = block.run(v, B * T, D)
        v = Fn.LayerNormFn.apply(v, self.ln_depth.weight, self.ln_depth.bias, False)
        return _linear(v, self.head.weight, None).view(B * T, D, -1)

    # ------------------------------------------------------------------------------------------ sampling
    @torch.no_grad()
    def sample(self, conds: torch.LongTensor, top_k: Optional[float] = None, top_p: Optional[float] = None,
               softmax_temperature: float = 1.0, use_fp16: bool = True) -> Tuple[torch.FloatTensor, torch.LongTensor]:
        """reference stage2/layers.py:397-477 -> (logits [B*T, D, vocab], codes [B, T, D]).  The filtering and the draw are the
        reference's torch calls; the steps run in libb200vq.so with one preallocated KV cache per layer per transformer (the
        depth caches are [B, D, C], reused at every position).  `use_fp16` is accepted and ignored, as in GPT.sample."""
        B, T, D, S = conds.shape[0], self.img_num_tokens, self.depth_num_tokens, self.vocab_img_size
        past = depth_past = codes = logits = None
        for i in range(T):
            if codes is None:
                hidden, past = self.sample_spatial_step(None, conds, None, use_fp16, None)
            else:
                hidden, past = self.sample_spatial_step(codes[:, -D:], conds, self.pos_emb_code[:, i - 1:i, :], use_fp16, past)
            last_len = 0 if codes is None else codes.shape[-1]
            for d in range(D):
                if d == 0:
                    logits_, depth_past = self.sample_depth_step(None, hidden, None, use_fp16, depth_past)
                else:
                    logits_, depth_past = self.sample_depth_step(codes[:, last_len:], hidden, self.pos_emb_depth[:, d - 1:d, :],
                                                                 use_fp16, depth_past)
                logits_ = logits_.to(dtype=torch.float32) / softmax_temperature
                idx = _filter_and_draw(logits_, top_k, top_p)
                codes = idx if codes is None else torch.cat([codes, idx], axis=1)
                logits = logits_ if logits is None else torch.cat([logits, logits_], axis=1)
        return logits.view(B * T, D, S), codes.view(B, T, D)

    def _heads(self, blocks) -> Tuple[int, int]:
        C = self.head.weight.shape[1]
        heads = blocks[0].attn.n_heads if len(blocks) else 1
        return heads, C // heads

    @torch.no_grad()
    def sample_spatial_step(self, codes, conds, pos_code, use_fp16: bool = True, past=None):
        """reference stage2/layers.py:479-512 -> (hidden [B, 1, C] = ln_spatial of the newest row, past).  codes: the previous
        position's D codes [B, D] (None on the first step), embedded as their sum over depth plus pos_code (:501-502).
        `past` is this implementation's cache object: per-layer key / value buffers [B, Tc + T, C] and the rows filled."""
        C = self.head.weight.shape[1]
        heads, hs = self._heads(self.spatial_transformer)
        if codes is None:
            assert past is None
            conds = conds.contiguous()
            B, Tc = conds.shape
            empty = torch.empty(B, 0, dtype=torch.int64, device=conds.device)
            x = ops.token_embed_fwd(conds, empty, self.tok_emb_cond.weight, self.pos_emb_cond.view(Tc, C), self.tok_emb_code.weight,
                                    self.pos_emb_code.view(-1, C))
            x, past = _cached_prefix(self.spatial_transformer, x, B, Tc, Tc + self.img_num_tokens, heads, hs)
            x = Fn.LayerNormFn.apply(x, self.ln_spatial.weight, self.ln_spatial.bias, False)
            x = ops.copy_rows(x, B, Tc, 1, Tc - 1, 0, 1)
        else:
            assert past is not None
            B = codes.shape[0]
            x = ops.code_sum_embed(codes, codes.shape[1], self.tok_emb_code.weight, pos_code.contiguous().view(C))
            x = _cached_step(self.spatial_transformer, x, past, heads, hs)
            x = Fn.LayerNormFn.apply(x, self.ln_spatial.weight, self.ln_spatial.bias, False)
        return x.view(B, 1, C), past

    @torch.no_grad()
    def sample_depth_step(self, codes, hidden, pos_depth, use_fp16: bool = True, past=None):
        """reference stage2/layers.py:514-547 -> (logits [B, vocab], past).  codes None: depth step 0 on `hidden`, with
        ln_depth applied twice (:531, :542); a `past` handed in then is a previous position's depth cache ([B, D, C] per
        layer), whose buffers are reused (step 0 writes row 0 and reads nothing beyond it).  Otherwise codes [B, d] are this position's codes so far,
        embedded as their sum plus pos_depth (:534-535)."""
        C = self.head.weight.shape[1]
        heads, hs = self._heads(self.depth_transformer)
        ln = lambda t: Fn.LayerNormFn.apply(t, self.ln_depth.weight, self.ln_depth.bias, False)   # noqa: E731
        if codes is None:
            x = hidden.contiguous().view(-1, C)
            if past is None:
                B = x.shape[0]
                past = {"k": [torch.zeros(B, self.depth_num_tokens, C, device=x.device) for _ in self.depth_transformer],
                        "v": [torch.zeros(B, self.depth_num_tokens, C, device=x.device) for _ in self.depth_transformer]}
            past["len"] = 0          # one token attending to itself: decode_attention at row 0
            x = ln(_cached_step(self.depth_transformer, x, past, heads, hs))
        else:
            assert past is not None
            x = ops.code_sum_embed(codes, codes.shape[1], self.tok_emb_code.weight, pos_depth.contiguous().view(C))
            x = _cached_step(self.depth_transformer, x, past, heads, hs)
        x = ln(x)
        return _linear(x, self.head.weight, None), past
