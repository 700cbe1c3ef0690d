"""autograd.Functions that stitch the C-ABI kernels into the forward/backward of the ViT blocks
and the quantiser.  Saved tensors were chosen for HBM footprint (SURVEY.md section 7 'Memory at
config 2'): LayerNorm statistics, one copy of qkv, the attention output and its log-sum-exp
(never the N x N probabilities), the tanh output.

Precision modes (`set_precision`, env B200VQ_PRECISION):

  "fp16"    default.  The four projections of every transformer block and their dgrad / wgrad run as
            f16 tensor-core GEMMs: operands are stored in fp16 by the kernel that produces them
            (LayerNorm, tanh epilogue, attention epilogue), accumulation / residual stream / LayerNorm /
            softmax / losses stay fp32.  fp16 has the same 11-bit significand as tf32, so the results
            carry tf32-level rounding at twice the tensor-core rate and half the operand traffic.
            Gradient operands are multiplied by a power of two S chosen on the device from the gradient
            entering each transformer stack (`ops.grad_scale`) and every fp32 result is multiplied by 1/S
            in the producing epilogue: exact, and it keeps fp16's exponent range out of the picture.
            The attention core takes fp16 operands as well (dim_head 64: the fp16 core; other head sizes on the tf32
            kernels from a tf32-rounded fp32 qkv matrix).
  "tf32"    every GEMM on tf32 tensor cores with operands rounded to nearest where they are produced
            (round 1's data path).
  "parity"  error-compensated 3xTF32 GEMMs and attention (fp32-grade, ~3-6x slower): the mode the
            reference-parity tests use to show margin against the 1e-3 tolerance.

`pre_quant` decides the code indices, so `QuantLinear` always runs it as 3xTF32 whatever the mode."""
from __future__ import annotations

import os
from typing import List, Optional, Sequence, Tuple

import torch
from torch.amp import custom_bwd, custom_fwd

from . import ops

# Under torch.autocast (the reference's `--use_amp`, main.py precision=16) the unchanged nn.Linear
# pre_quant / post_quant hand fp16 tensors to these Functions.  Every Function therefore declares
# fp32 inputs (custom_fwd casts, and disables autocast inside) -- the kernels' own mixed precision
# (tensor-core operands, fp32 accumulation / residual stream / statistics) is fixed by design.
_fwd = custom_fwd(device_type="cuda", cast_inputs=torch.float32)
_bwd = custom_bwd(device_type="cuda")

Tensor = torch.Tensor

# cta_group used for the big GEMMs (2 = CTA pair per 256-row tile); a module-level switch so
# that tests and bench.py can pin it
GEMM_CTA_GROUP = 2

PRECISIONS = ("fp16", "tf32", "parity")
_precision = os.environ.get("B200VQ_PRECISION", "fp16")
if _precision not in PRECISIONS:
    raise RuntimeError(f"B200VQ_PRECISION must be one of {PRECISIONS}, got {_precision!r}")


def set_precision(mode: str) -> str:
    """select the data path of subsequently *recorded* graphs; returns the previous mode"""
    global _precision
    if mode not in PRECISIONS:
        raise ValueError(f"precision must be one of {PRECISIONS}, got {mode!r}")
    prev, _precision = _precision, mode
    return prev


def get_precision() -> str:
    return _precision


# ------------------------------------------------------------------------------------------------
# weight shadows: the tensor-core copy of a parameter (tf32-rounded fp32, fp16, or the tf32 residue)
# ------------------------------------------------------------------------------------------------
_SHADOW_ATTR = "_b200vq_shadows"
_SHADOW_MAKERS = {"tf32": ops.round_tf32, "f16": ops.to_half, "lo": ops.split_tf32_lo}


def weight_shadow(w: Tensor, kind: str, in_backward: bool = False) -> Tensor:
    """Tensor-core copy of a parameter.  The copies hang off the parameter object itself (so they live
    and die with it -- a global cache keyed by address would hand a new parameter allocated at a recycled
    address the previous owner's values).

    Staleness: the cache key is (version counter, storage address).  In-place optimizer steps,
    ``load_state_dict`` and ``copy_`` bump the version; ``p.data = t`` moves the address.  Writes through
    ``p.data`` (EMA weight swaps, some init helpers) bump neither, so outside autograd recording -- where
    those swaps happen and no optimizer runs -- the shadow is simply recomputed on every call (0.1 ms for
    the whole base model), and `invalidate_shadows()` exists for the remaining case (a ``.data`` write
    between two grad-enabled forwards).  A refresh always writes a *new* buffer: the old one may be held
    by ``ctx.save_for_backward`` of a graph that has not run backward yet.  Backward nodes (`in_backward`) save
    the parameter itself, so autograd has already verified its version when they ask: the cached copy is valid
    there although gradient recording is off."""
    cache = getattr(w, _SHADOW_ATTR, None)
    key = (w._version, w.data_ptr())
    if cache is not None and (in_backward or torch.is_grad_enabled()):
        ent = cache.get(kind)
        if ent is not None and ent[0] == key and ent[1].device == w.device:
            return ent[1]
    src = w.detach()
    if not src.is_contiguous():
        src = src.contiguous()
    out = _SHADOW_MAKERS[kind](src)
    try:
        if cache is None:
            cache = {}
            setattr(w, _SHADOW_ATTR, cache)
        cache[kind] = (key, out)
    except AttributeError:      # exotic tensor subclasses without a __dict__: just do not cache
        pass
    return out


def tf32_shadow(w: Tensor) -> Tensor:
    return weight_shadow(w, "tf32")


def invalidate_shadows(module: torch.nn.Module) -> None:
    """Drop the cached shadows of every parameter of `module` (call after writing weights through
    ``p.data`` while autograd recording is on; every other way of changing a weight is detected)."""
    for p in module.parameters():
        if hasattr(p, _SHADOW_ATTR):
            delattr(p, _SHADOW_ATTR)


class _W:
    """operand view of one weight for the current precision: `.a` (+ `.lo` in parity mode)"""
    __slots__ = ("a", "lo")

    def __init__(self, w: Tensor, mode: str, in_backward: bool = False):
        if mode == "parity":
            src = w.detach()
            self.a = src if src.is_contiguous() else src.contiguous()
            self.lo = weight_shadow(w, "lo", in_backward)
        else:
            self.a = weight_shadow(w, "f16" if mode == "fp16" else "tf32", in_backward)
            self.lo = None


def _mm(a: Tensor, w: _W, M: int, N: int, K: int, mode: str, **kw) -> Tensor:
    """activation x weight GEMM of the fp32 data paths: tf32 (operands pre-rounded) or 3xTF32 (parity)"""
    if mode == "parity":
        kw.pop("round_out", None)
        return ops.gemm(a, w.a, M, N, K, a_lo=ops.split_tf32_lo(a), b_lo=w.lo, cta_group=GEMM_CTA_GROUP, **kw)
    return ops.gemm(a, w.a, M, N, K, cta_group=GEMM_CTA_GROUP, **kw)


def _wgrad(dy: Tensor, x: Tensor, rows: int, cols: int, mode: str = "tf32", inv_scale: Optional[Tensor] = None) -> Tensor:
    """dW[rows, cols] = dy[M, rows]^T . x[M, cols]   (both operands MN-major, split-K over the tokens)"""
    M = dy.shape[0]
    half = dy.dtype == torch.float16
    splits = ops.pick_splits(M, rows, cols, k_atom=64 if half else 32)
    kw = {}
    if mode == "parity":
        kw = dict(a_lo=ops.split_tf32_lo(dy), b_lo=ops.split_tf32_lo(x))
    if splits == 1:
        return ops.gemm(dy, x, rows, cols, M, a_major=1, b_major=1, cta_group=GEMM_CTA_GROUP, alpha=inv_scale if half else None, **kw)
    part = ops.gemm(dy, x, rows, cols, M // splits, a_major=1, b_major=1, splits=splits, cta_group=GEMM_CTA_GROUP, **kw)
    return ops.splitk_reduce(part, alpha=inv_scale if half else None)


GEMM_COLSUM = os.environ.get("B200VQ_GEMM_COLSUM", "1") != "0"   # bias-gradient column sums from the dgrad epilogue
_COLSUM_ATTR = "_b200vq_colsum"


def _attach_colsum(t: Tensor, colsum: Tensor) -> Tensor:
    """Remember the column sums of a gradient tensor the LayerNorm-backward kernel produced for free.
    The next backward node down the residual stream (the patch embedding) needs exactly colsum(t) for its
    bias gradient; it picks the value up with `_colsum_of` if (and only if) the very same, unmodified
    tensor reaches it, and recomputes otherwise."""
    setattr(t, _COLSUM_ATTR, (colsum, t._version, t.data_ptr()))
    return t


def _colsum_of(t: Tensor) -> Tensor:
    tag = getattr(t, _COLSUM_ATTR, None)
    if tag is not None:
        colsum, version, ptr = tag
        if version == t._version and ptr == t.data_ptr() and colsum.shape[0] == t.shape[-1]:
            return colsum
    return ops.colsum(t)


# ------------------------------------------------------------------------------------------------
# one pre-norm block: x -> attn(LN(x)) + x -> ff(LN(.)) + .   (reference layers.py:145-148 with :85-132)
# parameters per block, in order: ln1_w, ln1_b, w_qkv, w_out, b_out, ln2_w, ln2_b, w1, b1, w2, b2
# ------------------------------------------------------------------------------------------------
LAYER_PARAMS = 11
# The first and the last GEMM of the model (patch embedding, to_pixel: K or N = 192, memory-bound, 0.5 % of the FLOPs)
# always run as 3xTF32: their rounding is not averaged out by anything downstream (to_pixel writes the pixels the
# 1e-3 tolerance is measured on), and the extra passes cost ~1 ms per 250 ms step.
PRECISE_IO = os.environ.get("B200VQ_PRECISE_IO", "1") != "0"
ATTENTION_F16 = os.environ.get("B200VQ_ATTENTION_F16", "1") != "0"   # fp16 mode: fp16-operand attention core for dim_head 64
# Bit-reproducible backward on request: the codebook and token-embedding gradients are then summed in a fixed order
# instead of with float atomics (every other kernel of the path is deterministic already).  B200VQ_DETERMINISTIC=1, or
# torch.use_deterministic_algorithms(True), checked when the backward runs.
DETERMINISTIC = os.environ.get("B200VQ_DETERMINISTIC", "0") == "1"


def deterministic() -> bool:
    return DETERMINISTIC or torch.are_deterministic_algorithms_enabled()


def f16_supported(dim: int, inner: int, mlp: int) -> bool:
    """the fp16 GEMMs read whole 64-element atoms of every MN-major operand (wgrad, dgrad)"""
    return dim % 64 == 0 and inner % 64 == 0 and mlp % 64 == 0


def _block_fwd_fp32(x, prm, dims, mode):
    """tf32 / parity data path: every tensor fp32"""
    ln1_w, ln1_b, w_qkv, w_out, b_out, ln2_w, ln2_b, w1, b1, w2, b2 = prm
    B, N, heads, dh = dims
    M, D = x.shape
    inner, mlp, scale = heads * dh, w1.shape[0], dh ** -0.5
    rnd = mode == "tf32"
    wq, wo, w1s, w2s = (_W(w, mode) for w in (w_qkv, w_out, w1, w2))
    h1, mean1, rstd1 = ops.layernorm_fwd(x, ln1_w, ln1_b, rnd)
    qkv = _mm(h1, wq, M, 3 * inner, D, mode, round_out=rnd)
    if mode == "parity":
        o, lse = ops.attention_exact_fwd(qkv, B, N, heads, dh, scale)
    else:
        o, lse = ops.attention_fwd(qkv, B, N, heads, dh, scale, True)
    x1 = _mm(o, wo, M, D, inner, mode, bias=b_out, res=x)
    h2, mean2, rstd2 = ops.layernorm_fwd(x1, ln2_w, ln2_b, rnd)
    t = _mm(h2, w1s, M, mlp, D, mode, bias=b1, act=1, round_out=rnd)
    x2 = _mm(t, w2s, M, D, mlp, mode, bias=b2, res=x1)
    return x2, (x, mean1, rstd1, h1, qkv, o, lse, x1, mean2, rstd2, h2, t)


def _block_bwd_fp32(saved, prm, dims, mode, g, g_colsum, need_w):
    x, mean1, rstd1, h1, qkv, o, lse, x1, mean2, rstd2, h2, t = saved
    ln1_w, _, w_qkv, w_out, _, ln2_w, _, w1, _, w2, _ = prm
    B, N, heads, dh = dims
    M, D = x.shape
    inner, mlp, scale = heads * dh, w1.shape[0], dh ** -0.5
    rnd = mode == "tf32"
    wq, wo, w1s, w2s = (_W(w, mode, True) for w in (w_qkv, w_out, w1, w2))
    # ---- feed-forward branch
    db2 = (g_colsum if g_colsum is not None else ops.colsum(g)) if need_w else None
    dw2 = _wgrad(g, t, D, mlp, mode) if need_w else None
    db1 = None
    if GEMM_COLSUM and need_w:
        dt, db1 = _mm(g, w2s, M, mlp, D, mode, b_major=1, aux=t, round_out=rnd, want_colsum=True)   # (g W2) * (1 - t^2), colsum(dt)
    else:
        dt = _mm(g, w2s, M, mlp, D, mode, b_major=1, aux=t, round_out=rnd)
        if need_w:
            db1 = ops.colsum(dt)
    dw1 = _wgrad(dt, h2, mlp, D, mode) if need_w else None
    dh2 = _mm(dt, w1s, M, D, mlp, mode, b_major=1)
    del dt
    g1, dln2_w, dln2_b, dbo = ops.layernorm_bwd(dh2, x1, mean2, rstd2, ln2_w, g, want_colsum=True)
    del dh2
    # ---- attention branch (dbo = colsum(g1) came with the kernel above)
    dwo = _wgrad(g1, o, D, inner, mode) if need_w else None
    do = _mm(g1, wo, M, inner, D, mode, b_major=1, round_out=rnd)
    if mode == "parity":
        dqkv = ops.attention_exact_bwd(qkv, o, lse, do, B, N, heads, dh, scale)
    else:
        dqkv = ops.attention_bwd(qkv, o, lse, do, B, N, heads, dh, scale, True)
    del do
    dwq = _wgrad(dqkv, h1, 3 * inner, D, mode) if need_w else None
    dh1 = _mm(dqkv, wq, M, D, 3 * inner, mode, b_major=1)
    del dqkv
    gx, dln1_w, dln1_b, gx_sum = ops.layernorm_bwd(dh1, x, mean1, rstd1, ln1_w, g1, want_colsum=True)
    grads = (dln1_w, dln1_b, dwq, dwo, dbo, dln2_w, dln2_b, dw1, db1, dw2, db2) if need_w else (None,) * LAYER_PARAMS
    return gx, gx_sum, None, grads


def _block_fwd_f16(x, prm, dims):
    """fp16-operand data path: residual stream x / x1 / x2 and qkv fp32, every other GEMM operand fp16"""
    ln1_w, ln1_b, w_qkv, w_out, b_out, ln2_w, ln2_b, w1, b1, w2, b2 = prm
    B, N, heads, dh = dims
    M, D = x.shape
    inner, mlp, scale = heads * dh, w1.shape[0], dh ** -0.5
    cg = GEMM_CTA_GROUP
    wq, wo, w1h, w2h = (weight_shadow(w, "f16") for w in (w_qkv, w_out, w1, w2))
    h1, mean1, rstd1 = ops.layernorm_fwd(x, ln1_w, ln1_b, False, out_half=True)
    if dh == 64 and ATTENTION_F16:
        qkv = ops.gemm(h1, wq, M, 3 * inner, D, out_half=True, cta_group=cg)              # fp16 qkv -> fp16 attention core
        o, lse = ops.attention_f16_fwd(qkv, B, N, heads, dh, scale)
    else:
        qkv = ops.gemm(h1, wq, M, 3 * inner, D, round_out=True, cta_group=cg)             # fp32, tf32-rounded: tf32 attention core
        o, lse = ops.attention_fwd(qkv, B, N, heads, dh, scale, False, out_half=True)
    x1 = ops.gemm(o, wo, M, D, inner, bias=b_out, res=x, cta_group=cg)
    h2, mean2, rstd2 = ops.layernorm_fwd(x1, ln2_w, ln2_b, False, out_half=True)
    t = ops.gemm(h2, w1h, M, mlp, D, bias=b1, act=1, out_half=True, cta_group=cg)
    x2 = ops.gemm(t, w2h, M, D, mlp, bias=b2, res=x1, cta_group=cg)
    return x2, (x, mean1, rstd1, h1, qkv, o, lse, x1, mean2, rstd2, h2, t)


def _block_bwd_f16(saved, prm, dims, g, g_colsum, gh, sc, need_w):
    """g: fp32 gradient of the block output; gh = fp16(g * S); sc = device tensor [S, 1/S]"""
    x, mean1, rstd1, h1, qkv, o, lse, x1, mean2, rstd2, h2, t = saved
    ln1_w, _, w_qkv, w_out, _, ln2_w, _, w1, _, w2, _ = prm
    B, N, heads, dh = dims
    M, D = x.shape
    inner, mlp, scale = heads * dh, w1.shape[0], dh ** -0.5
    cg = GEMM_CTA_GROUP
    S, inv = sc[0:1], sc[1:2]
    wq, wo, w1h, w2h = (weight_shadow(w, "f16", True) for w in (w_qkv, w_out, w1, w2))
    # ---- feed-forward branch
    db2 = (g_colsum if g_colsum is not None else ops.colsum(g)) if need_w else None
    dw2 = _wgrad(gh, t, D, mlp, inv_scale=inv) if need_w else None
    db1 = None
    if need_w:
        dt, db1 = ops.gemm(gh, w2h, M, mlp, D, b_major=1, aux=t, out_half=True, cta_group=cg, want_colsum=True)   # still carries S
        db1 = db1 * inv
    else:
        dt = ops.gemm(gh, w2h, M, mlp, D, b_major=1, aux=t, out_half=True, cta_group=cg)
    dw1 = _wgrad(dt, h2, mlp, D, inv_scale=inv) if need_w else None
    dh2 = ops.gemm(dt, w1h, M, D, mlp, b_major=1, out_half=True, cta_group=cg)                      # fp16, carries S
    del dt
    g1, dln2_w, dln2_b, dbo, g1h = ops.layernorm_bwd(dh2, x1, mean2, rstd2, ln2_w, g, want_colsum=True, half_scale=S, dy_scale=inv)
    del dh2
    # ---- attention branch
    dwo = _wgrad(g1h, o, D, inner, inv_scale=inv) if need_w else None
    if qkv.dtype == torch.float16:
        do = ops.gemm(g1h, wo, M, inner, D, b_major=1, out_half=True, cta_group=cg)                # fp16, still carries S
        dqkv = ops.attention_f16_bwd(qkv, o, lse, do, B, N, heads, dh, scale)                      # fp16, carries S
    else:
        do = ops.gemm(g1h, wo, M, inner, D, b_major=1, alpha=inv, round_out=True, cta_group=cg)
        dqkv = ops.attention_bwd(qkv, o, lse, do, B, N, heads, dh, scale, False, half_scale=S)     # fp16, carries S
    del g1h, do
    dwq = _wgrad(dqkv, h1, 3 * inner, D, inv_scale=inv) if need_w else None
    dh1 = ops.gemm(dqkv, wq, M, D, 3 * inner, b_major=1, out_half=True, cta_group=cg)               # fp16, carries S
    del dqkv
    gx, dln1_w, dln1_b, gx_sum, gxh = ops.layernorm_bwd(dh1, x, mean1, rstd1, ln1_w, g1, want_colsum=True, half_scale=S, dy_scale=inv)
    grads = (dln1_w, dln1_b, dwq, dwo, dbo, dln2_w, dln2_b, dw1, db1, dw2, db2) if need_w else (None,) * LAYER_PARAMS
    return gx, gx_sum, gxh, grads


_SAVED_PER_BLOCK = 12


class TransformerFn(torch.autograd.Function):
    """`depth` pre-norm blocks followed by the final LayerNorm (reference layers.py:135-150) as ONE autograd
    node: the hand-off between blocks in backward (the residual gradient, its column sums, its fp16 copy and
    the gradient scale) is plain Python, not something autograd has to carry between nodes.

    apply(x [M, D], B, N, heads, dh, round_final, norm_w, norm_b, *block_params)"""

    @staticmethod
    @_fwd
    def forward(ctx, x, B, N, heads, dh, round_final, norm_w, norm_b, *prm):
        depth = len(prm) // LAYER_PARAMS
        M, D = x.shape
        dims = (B, N, heads, dh)
        mode = _precision
        if mode == "fp16" and not (depth and f16_supported(D, heads * dh, prm[7].shape[0])):
            mode = "tf32"
        saved: List[Tensor] = []
        h = x
        for i in range(depth):
            p = prm[i * LAYER_PARAMS:(i + 1) * LAYER_PARAMS]
            h, sv = _block_fwd_f16(h, p, dims) if mode == "fp16" else _block_fwd_fp32(h, p, dims, mode)
            saved.extend(sv)
        y, mean, rstd = ops.layernorm_fwd(h, norm_w, norm_b, bool(round_final) and mode != "parity" and not PRECISE_IO)
        ctx.save_for_backward(h, mean, rstd, norm_w, *prm, *saved)
        ctx.cfg = (dims, depth, mode)
        return y

    @staticmethod
    @_bwd
    def backward(ctx, gy):
        dims, depth, mode = ctx.cfg
        h, mean, rstd, norm_w = ctx.saved_tensors[:4]
        prm = ctx.saved_tensors[4:4 + depth * LAYER_PARAMS]
        saved = ctx.saved_tensors[4 + depth * LAYER_PARAMS:]
        g, dnorm_w, dnorm_b, g_sum = ops.layernorm_bwd(gy.contiguous(), h, mean, rstd, norm_w, None, want_colsum=True)
        gh = sc = None
        if mode == "fp16" and depth:
            # The gradient scale of this stack, from the gradient that actually enters it: S puts max|g| at 2^6,
            # leaving ~2^10 of headroom below fp16's 65504 for whatever the blocks amplify and full 11-bit
            # precision down to 2^-20 of max|g| (saturating conversions are the backstop).
            sc = ops.grad_scale(g)
            gh = ops.to_half(g, sc[0:1])
        grads: List[Optional[Tensor]] = [None] * (depth * LAYER_PARAMS)
        for i in reversed(range(depth)):
            p = prm[i * LAYER_PARAMS:(i + 1) * LAYER_PARAMS]
            sv = saved[i * _SAVED_PER_BLOCK:(i + 1) * _SAVED_PER_BLOCK]
            # Parameter gradients are all-or-nothing per block: a frozen stage-1 model (reference
            # stage2/transformer.py:44-46) or torch.autograd.grad w.r.t. another tensor skips the four wgrad
            # GEMMs and the bias column sums.
            need_w = any(ctx.needs_input_grad[8 + i * LAYER_PARAMS:8 + (i + 1) * LAYER_PARAMS])
            if mode == "fp16":
                g, g_sum, gh, gr = _block_bwd_f16(sv, p, dims, g, g_sum, gh, sc, need_w)
            else:
                g, g_sum, _, gr = _block_bwd_fp32(sv, p, dims, mode, g, g_sum, need_w)
            grads[i * LAYER_PARAMS:(i + 1) * LAYER_PARAMS] = gr
        _attach_colsum(g, g_sum)
        return (g, None, None, None, None, None, dnorm_w, dnorm_b, *grads)


class LayerNormFn(torch.autograd.Function):
    """nn.LayerNorm(dim) stand-alone (PreNorm called outside the fused stack; reference layers.py:85-92)"""

    @staticmethod
    @_fwd
    def forward(ctx, x, w, b, round_out):
        y, mean, rstd = ops.layernorm_fwd(x, w, b, bool(round_out))
        ctx.save_for_backward(x, mean, rstd, w)
        return y

    @staticmethod
    @_bwd
    def backward(ctx, g):
        x, mean, rstd, w = ctx.saved_tensors
        dx, dw, db, dx_sum = ops.layernorm_bwd(g.contiguous(), x, mean, rstd, w, None, want_colsum=True)
        _attach_colsum(dx, dx_sum)
        return dx, dw, db, None


class LinearFn(torch.autograd.Function):
    """y = act(x W^T + b): stand-alone GEMM unit used by the sub-modules when they are called outside the
    fused stack (reference layers.py:99-101,118,120) and by QuantLinear (vitvqgan.py:38-39).
    precise=True forces the 3xTF32 product whatever the global mode."""

    @staticmethod
    @_fwd
    def forward(ctx, x, w, b, act, precise):
        M, K = x.shape
        N = w.shape[0]
        mode = "parity" if (precise or _precision == "parity") else "tf32"
        xr = x if mode == "parity" else ops.round_tf32(x)
        y = _mm(xr, _W(w, mode), M, N, K, mode, bias=b, act=int(act))
        ctx.save_for_backward(xr, w, y if act else None)
        ctx.cfg = (b is not None, mode)
        return y

    @staticmethod
    @_bwd
    def backward(ctx, g):
        xr, w, y = ctx.saved_tensors
        has_bias, mode = ctx.cfg
        M, K = xr.shape
        N = w.shape[0]
        g = g.contiguous()
        if y is not None:   # tanh backward folded into the dgrad epilogue is only available fused
            g = g * (1 - y * y)
        gr = g if mode == "parity" else ops.round_tf32(g)
        need_x, need_w, need_b = ctx.needs_input_grad[:3]
        db = ops.colsum(gr) if (has_bias and need_b) else None
        dw = _wgrad(gr, xr, N, K, mode) if need_w else None
        dx = _mm(gr, _W(w, mode, True), M, K, N, mode, b_major=1) if need_x else None
        return dx, dw, db, None, None


class LinearPosFn(torch.autograd.Function):
    """x W^T + b + table[row % n_tok]: ``post_quant`` with the decoder's positional table added in the GEMM epilogue
    (reference vitvqgan.py:69 followed by layers.py:210) -- SURVEY.md section 8f-1: the [M, D] tensor between the two
    is never written.  Always 3xTF32, like `QuantLinear`."""

    @staticmethod
    @_fwd
    def forward(ctx, x, w, b, table):
        M, K = x.shape
        N = w.shape[0]
        n_tok = table.numel() // N
        y = _mm(x, _W(w, "parity"), M, N, K, "parity", bias=b, res=table.view(n_tok, N), res_row_mod=n_tok)
        ctx.save_for_backward(x, w)
        ctx.has_bias = b is not None
        return y

    @staticmethod
    @_bwd
    def backward(ctx, g):
        x, w = ctx.saved_tensors
        M, K = x.shape
        N = w.shape[0]
        g = g.contiguous()
        need_x, need_w, need_b = ctx.needs_input_grad[:3]
        db = _colsum_of(g) if (ctx.has_bias and need_b) else None
        dw = _wgrad(g, x, N, K, "parity") if need_w else None
        dx = _mm(g, _W(w, "parity", True), M, K, N, "parity", b_major=1) if need_x else None
        return dx, dw, db, None


class AttentionCoreFn(torch.autograd.Function):
    """softmax(q k^T * scale) v on the packed qkv matrix (reference layers.py:124-130), stand-alone"""

    @staticmethod
    @_fwd
    def forward(ctx, qkv, B, N, heads, dh):
        scale = dh ** -0.5
        exact = _precision == "parity"
        if exact:
            qr = qkv
            o, lse = ops.attention_exact_fwd(qr, B, N, heads, dh, scale)
        else:
            qr = ops.round_tf32(qkv)
            o, lse = ops.attention_fwd(qr, B, N, heads, dh, scale, False)
        ctx.save_for_backward(qr, o, lse)
        ctx.dims = (B, N, heads, dh, exact)
        return o

    @staticmethod
    @_bwd
    def backward(ctx, g):
        qr, o, lse = ctx.saved_tensors
        B, N, heads, dh, exact = ctx.dims
        if exact:
            dqkv = ops.attention_exact_bwd(qr, o, lse, g.contiguous(), B, N, heads, dh, dh ** -0.5)
        else:
            dqkv = ops.attention_bwd(qr, o, lse, ops.round_tf32(g.contiguous()), B, N, heads, dh, dh ** -0.5, False)
        return dqkv, None, None, None, None


class PatchEmbedFn(torch.autograd.Function):
    """Conv2d(C, D, k=s=p) + 'b c h w -> b (h w) c' + positional table
    (reference layers.py:168-172,178-179) as one GEMM over the im2col view."""

    @staticmethod
    @_fwd
    def forward(ctx, img, w, b, pos, p):
        B, C, H, W = img.shape
        D = w.shape[0]
        ph, pw = ops._pair(p)
        n_tok = (H // ph) * (W // pw)
        mode = "parity" if (PRECISE_IO or _precision == "parity") else "tf32"
        patches = ops.patchify(img, p, mode == "tf32")
        M, pd = patches.shape
        ws = _W(w, mode)
        ws.a = ws.a.view(D, pd)
        if ws.lo is not None:
            ws.lo = ws.lo.view(D, pd)
        x = _mm(patches, ws, M, D, pd, mode, bias=b, res=pos.view(n_tok, D), res_row_mod=n_tok)
        ctx.save_for_backward(patches, w)
        ctx.geom = (B, C, H, W, p, mode)
        return x

    @staticmethod
    @_bwd
    def backward(ctx, g):
        patches, w = ctx.saved_tensors
        B, C, H, W, p, mode = ctx.geom
        D = w.shape[0]
        M, pd = patches.shape
        g = g.contiguous()
        db = _colsum_of(g) if ctx.needs_input_grad[2] else None
        dw = _wgrad(g, patches, D, pd, mode).view_as(w) if ctx.needs_input_grad[1] else None
        dimg = None
        if ctx.needs_input_grad[0]:
            ws = _W(w, mode, True)
            ws.a = ws.a.view(D, pd)
            if ws.lo is not None:
                ws.lo = ws.lo.view(D, pd)
            dpat = _mm(g, ws, M, pd, D, mode, b_major=1)
            dimg = ops.unpatchify(dpat, None, B, C, H, W, p)
        return dimg, dw, db, None, None


class ToPixelFn(torch.autograd.Function):
    """'b (h w) c -> b c h w' + ConvTranspose2d(D, C, k=s=p) (reference layers.py:202-205,212)
    as one GEMM plus a pixel-shuffle store."""

    @staticmethod
    @_fwd
    def forward(ctx, x, w, b, B, H, W, p):
        M, D = x.shape
        C = w.shape[1]
        ph, pw = ops._pair(p)
        pd = C * ph * pw
        mode = "parity" if (PRECISE_IO or _precision == "parity") else "tf32"
        ws = _W(w, mode)
        ws.a = ws.a.view(D, pd)
        if ws.lo is not None:
            ws.lo = ws.lo.view(D, pd)
        y = _mm(x, ws, M, pd, D, mode, b_major=1)
        img = ops.unpatchify(y, b, B, C, H, W, p)
        ctx.save_for_backward(x, w)
        ctx.geom = (B, C, H, W, p, mode)
        return img

    @staticmethod
    @_bwd
    def backward(ctx, g):
        x, w = ctx.saved_tensors
        B, C, H, W, p, mode = ctx.geom
        M, D = x.shape
        ph, pw = ops._pair(p)
        pd = C * ph * pw
        # the reference's adaptive GAN weight calls torch.autograd.grad(loss, get_last_layer()) twice per step
        # (vqperceptual.py:97-98): only dw is wanted there, so every product is guarded
        need_x, need_w, need_b = ctx.needs_input_grad[:3]
        dy = ops.patchify(g.contiguous(), p, mode == "tf32")
        db = ops.colsum(dy).view(C, ph * pw).sum(dim=1) if need_b else None
        dw = _wgrad(x, dy, D, pd, mode).view_as(w) if need_w else None
        dx = None
        if need_x:
            ws = _W(w, mode, True)
            ws.a = ws.a.view(D, pd)
            if ws.lo is not None:
                ws.lo = ws.lo.view(D, pd)
            dx = _mm(dy, ws, M, D, pd, mode)
        return dx, dw, db, None, None, None, None


class AddPosFn(torch.autograd.Function):
    """token + de_pos_embedding (reference layers.py:210)"""

    @staticmethod
    @_fwd
    def forward(ctx, x, pos):
        return ops.add_rows_mod(x, pos)

    @staticmethod
    @_bwd
    def backward(ctx, g):
        return g, None


class AddFn(torch.autograd.Function):
    """a + b on the residual stream (reference layers.py:147-148) for the unfused fallback path"""

    @staticmethod
    @_fwd
    def forward(ctx, a, b):
        flat = a.contiguous().view(-1, a.shape[-1])
        return ops.add_rows_mod(flat, b.contiguous().view(-1, a.shape[-1])).view_as(a)

    @staticmethod
    @_bwd
    def backward(ctx, g):
        return g, g


class VectorQuantizeFn(torch.autograd.Function):
    """BaseQuantizer.forward + VectorQuantizer.quantize (reference quantizers.py:38-63,74-92)."""

    @staticmethod
    @_fwd
    def forward(ctx, z, E, depth, beta, residual, use_norm):
        out, loss, idx = ops.vq_fwd(z, E, depth, beta, use_norm)
        ctx.save_for_backward(z, E, idx)
        ctx.cfg = (depth, beta, residual, use_norm)
        ctx.mark_non_differentiable(idx)
        return out, loss, idx

    @staticmethod
    @_bwd
    def backward(ctx, g_out, g_loss, _g_idx):
        z, E, idx = ctx.saved_tensors
        depth, beta, residual, use_norm = ctx.cfg
        if g_out is not None:
            g_out = g_out.contiguous()
        if g_loss is not None:
            g_loss = g_loss.contiguous()
        bwd = ops.vq_bwd_deterministic if deterministic() else ops.vq_bwd
        gz, gE = bwd(z, E, idx, g_out, g_loss, residual, beta, use_norm)
        return gz, gE, None, None, None, None


class EMAVectorQuantizeFn(torch.autograd.Function):
    """EMAVectorQuantizer's lookup: the forward of VectorQuantizeFn with the EMA loss and, with `stats`, the flat per-code
    statistics (non-differentiable).  E must be the codebook as it is at this forward and must not change before backward
    (EMAVectorQuantizer passes a copy when an update follows).  The codebook gets no gradient."""

    @staticmethod
    @_fwd
    def forward(ctx, z, E, depth, beta, residual, use_norm, stats):
        out, loss, idx, buf = ops.vq_fwd_ema(z, E, depth, beta, use_norm, stats, deterministic())
        ctx.save_for_backward(z, E, idx)
        ctx.cfg = (beta, residual, use_norm)
        if buf is None:
            ctx.mark_non_differentiable(idx)
            return out, loss, idx
        ctx.mark_non_differentiable(idx, buf)
        return out, loss, idx, buf

    @staticmethod
    @_bwd
    def backward(ctx, g_out, g_loss, _g_idx, _g_stats=None):
        z, E, idx = ctx.saved_tensors
        beta, residual, use_norm = ctx.cfg
        if residual:
            # the residual is built from z.detach() (quantizers.py:43): only the straight-through value reaches z
            gz = g_out
        else:
            # d(beta * mean((sg(q) - norm(z))^2))/dz is exactly vq_bwd's gz (its codebook term only ever reached E);
            # gz does not depend on how vq_bwd sums its codebook gradient, which is discarded here
            gz, _ = ops.vq_bwd(z, E, idx, None if g_out is None else g_out.contiguous(),
                               None if g_loss is None else g_loss.contiguous(), False, beta, use_norm)
        return gz, None, None, None, None, None, None
