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
head size ``embed_dim // n_heads`` must be 32 or 64, ``embed_dim`` <= 2048, ``vocab_img_size`` % 64 == 0 (the YAML's 6144 / 16 = 384-wide heads --
a 10.9 B-parameter model that cannot train under replicated fp32 DDP anyway, SURVEY.md section 8f-3 -- are not covered).

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


def _check_kernel_limits(embed_dim: int, n_heads: int) -> None:
    assert embed_dim % n_heads == 0
    hs = embed_dim // n_heads
    if hs not in (32, 64):
        raise NotImplementedError(f"b200vq stage 2: head size embed_dim // n_heads must be 32 or 64 (got {hs}); "
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
            idx = torch.multinomial(probs, num_samples=1).clone().detach()
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
        scale = 1.0 / math.sqrt(hs)
        if codes is None:
            assert past is None
            conds = conds.contiguous()
            B, Tc = conds.shape
            ctx = Tc + self.img_num_tokens
            dev = self.head.weight.device
            empty = torch.empty(B, 0, dtype=torch.int64, device=dev)
            x = ops.token_embed_fwd(conds, empty, self.tok_emb_cond.weight, self.pos_emb_cond.view(Tc, C),
                                    self.tok_emb_code.weight, self.pos_emb_code.view(-1, C))
            past = {"k": [], "v": [], "len": Tc}
            for block in self.blocks:
                att = block.attn
                h = Fn.LayerNormFn.apply(x, block.ln1.weight, block.ln1.bias, False)
                mixed = ops.time_mix_fwd(h, att.time_mix.view(-1), Tc)
                w, b = att.packed_qkv()
                qkv = _linear(mixed, w, b)
                ck = torch.zeros(B, ctx, C, device=dev)
                cv = torch.zeros(B, ctx, C, device=dev)
                q3 = qkv.view(B, Tc, 3, C)
                ck[:, :Tc] = q3[:, :, 1]
                cv[:, :Tc] = q3[:, :, 2]
                past["k"].append(ck)
                past["v"].append(cv)
                o = CausalAttentionFn.apply(qkv, B, Tc, heads, hs, Tc)      # the condition prefix sees itself fully (:83-85 with T == cond_len)
                x = _linear(o, att.proj.weight, att.proj.bias, x)
                x = block.mlp.core(Fn.LayerNormFn.apply(x, block.ln2.weight, block.ln2.bias, False), res=x)
            x = Fn.LayerNormFn.apply(x, self.layer_norm.weight, self.layer_norm.bias, False)
            x = ops.copy_rows(x, B, Tc, 1, Tc - 1, 0, 1)
        else:
            assert past is not None
            B = codes.shape[0]
            pos = past["len"]
            # a one-token sequence: time_shift(x) is all zeros (reference :58 on T == 1), so the mix is x * time_mix + 0
            x = ops.token_embed_fwd(torch.empty(B, 0, dtype=torch.int64, device=codes.device), codes.contiguous().view(B, 1),
                                    self.tok_emb_cond.weight, self.pos_emb_cond.view(-1, C), self.tok_emb_code.weight,
                                    pos_code.contiguous().view(1, C))
            for li, block in enumerate(self.blocks):
                att = block.attn
                h = Fn.LayerNormFn.apply(x, block.ln1.weight, block.ln1.bias, False)
                mixed = ops.time_mix_fwd(h, att.time_mix.view(-1), 1)
                w, b = att.packed_qkv()
                qkv = _linear(mixed, w, b)
                o = ops.decode_attention(qkv, past["k"][li], past["v"][li], heads, hs, pos, scale)
                x = _linear(o, att.proj.weight, att.proj.bias, x)
                x = block.mlp.core(Fn.LayerNormFn.apply(x, block.ln2.weight, block.ln2.bias, False), res=x)
            past["len"] = pos + 1
            x = Fn.LayerNormFn.apply(x, self.layer_norm.weight, self.layer_norm.bias, False)
        logits = _linear(x, self.head.weight, None)
        return logits, past
