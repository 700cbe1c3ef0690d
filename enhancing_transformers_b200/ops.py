"""Tensor-level wrappers over the C ABI (include/b200vq.h).  PyTorch is plumbing here: it owns
device memory (caching allocator) and the current stream; every FLOP below runs in
libb200vq.so.  CPU tensors are rejected -- there is no CPU path."""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from . import _lib

Tensor = torch.Tensor


def _req(t: Optional[Tensor], name: str, dtype=torch.float32) -> None:
    if t is None:
        return
    if not t.is_cuda:
        raise RuntimeError(f"b200vq: `{name}` is on {t.device}; this implementation has no CPU path "
                           "(use the reference modules on CPU)")
    if t.dtype != dtype:
        raise RuntimeError(f"b200vq: `{name}` must be {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise RuntimeError(f"b200vq: `{name}` must be contiguous")
    if t.device.index != torch.cuda.current_device():
        # kernels launch on the current device's current stream: a tensor living elsewhere would be
        # dereferenced on the wrong GPU (one process per GPU is the supported layout, INTEGRATION.md)
        raise RuntimeError(f"b200vq: `{name}` lives on {t.device} but the current CUDA device is "
                           f"cuda:{torch.cuda.current_device()}; call torch.cuda.set_device (or use "
                           "`with torch.cuda.device_of(x):`) before invoking the module")


def _p(t: Optional[Tensor]):
    return None if t is None else t.data_ptr()


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def launch_count() -> int:
    return int(_lib.lib().b200vq_launch_count())


def set_sm_limit(n: int) -> None:
    """cap the persistent GEMM / attention grids at n CTAs (0 = all SMs): leaves SMs to a concurrent NCCL kernel"""
    _lib.lib().b200vq_set_sm_limit(int(n))


_HALF = torch.float16


def _req_any(t: Optional[Tensor], name: str) -> None:
    _req(t, name, t.dtype if t is not None and t.dtype in (torch.float32, _HALF) else torch.float32)


# ------------------------------------------------------------------------------------------ GEMM
def gemm(a: Tensor, b: Tensor, M: int, N: int, K: int, *, a_major: int = 0, b_major: int = 0,
         lda: Optional[int] = None, ldb: Optional[int] = None, out: Optional[Tensor] = None,
         bias: Optional[Tensor] = None, res: Optional[Tensor] = None, res_row_mod: int = 0,
         aux: Optional[Tensor] = None, act: int = 0, round_out: bool = False, splits: int = 1,
         cta_group: int = 1, bn: int = 0, want_colsum: bool = False, a_lo: Optional[Tensor] = None,
         b_lo: Optional[Tensor] = None, out_half: bool = False, alpha: Optional[Tensor] = None):
    """C[M,N] = epilogue(alpha * A . B^T).  See include/b200vq.h.  With splits > 1 returns [splits, M, N].
    The operand dtype picks the tensor-core flavour: fp32 -> b200vq_gemm_tf32 (or, with a_lo/b_lo, the
    error-compensated b200vq_gemm_3xtf32), fp16 -> b200vq_gemm_f16 (out_half: fp16 C; alpha: device scalar).
    want_colsum: also return colsum(C) (-> (C, colsum)); the epilogue emits per-16-row partial sums."""
    half = a.dtype == _HALF
    _req(a, "a", a.dtype if half else torch.float32); _req(b, "b", a.dtype)
    _req(bias, "bias"); _req(res, "res"); _req(alpha, "alpha")
    if aux is not None:
        _req(aux, "aux", _HALF if out_half else torch.float32)
    if lda is None:
        lda = a.shape[-1]
    if ldb is None:
        ldb = b.shape[-1]
    if out is None:
        out = torch.empty((splits, M, N) if splits > 1 else (M, N), device=a.device, dtype=_HALF if out_half else torch.float32)
    _req(out, "out", _HALF if out_half else torch.float32)
    part = torch.empty((M + 15) // 16, N, device=a.device, dtype=torch.float32) if want_colsum else None
    L = _lib.lib()
    ldres = res.shape[-1] if res is not None else 0
    ldaux = aux.shape[-1] if aux is not None else 0
    if half:
        if a_lo is not None or b_lo is not None:
            raise RuntimeError("b200vq: the 3xTF32 product takes fp32 operands")
        rc = L.b200vq_gemm_f16(_p(a), lda, a_major, _p(b), ldb, b_major, _p(out), N, int(out_half), M, N, K, splits, M * N,
                               _p(bias), _p(res), ldres, res_row_mod, _p(aux), ldaux, _p(part), act, int(round_out), _p(alpha),
                               cta_group, bn, _stream())
        _lib.check(rc, "gemm_f16")
    elif a_lo is not None:
        _req(a_lo, "a_lo"); _req(b_lo, "b_lo")
        if out_half or alpha is not None:
            raise RuntimeError("b200vq: fp16 output / alpha belong to the fp16 GEMM")
        rc = L.b200vq_gemm_3xtf32(_p(a), _p(a_lo), lda, a_major, _p(b), _p(b_lo), ldb, b_major, _p(out), N, M, N, K, splits,
                                  M * N, _p(bias), _p(res), ldres, res_row_mod, _p(aux), ldaux, _p(part), act, cta_group, bn,
                                  _stream())
        _lib.check(rc, "gemm_3xtf32")
    else:
        if out_half or alpha is not None:
            raise RuntimeError("b200vq: fp16 output / alpha belong to the fp16 GEMM")
        rc = L.b200vq_gemm_tf32(_p(a), lda, a_major, _p(b), ldb, b_major, _p(out), N, M, N, K, splits, M * N,
                                _p(bias), _p(res), ldres, res_row_mod, _p(aux), ldaux, _p(part), act, int(round_out),
                                cta_group, bn, _stream())
        _lib.check(rc, "gemm_tf32")
    if want_colsum:
        return out, colsum(part)
    return out


def splitk_reduce(part: Tensor, out: Optional[Tensor] = None, alpha: Optional[Tensor] = None) -> Tensor:
    _req(part, "part"); _req(alpha, "alpha")
    splits = part.shape[0]
    n = part[0].numel()
    if out is None:
        out = torch.empty(part.shape[1:], device=part.device, dtype=torch.float32)
    _lib.check(_lib.lib().b200vq_splitk_reduce(_p(part), splits, n, n, _p(alpha), _p(out), _stream()), "splitk_reduce")
    return out


# Output tile (rows, columns) of the persistent GEMM (csrc/gemm_tc.cu: kBM, kBNHalf, and the tf32 kinds' 128-column
# tile), keyed by the k-block width in elements (64: fp16, 32: tf32): the wave model of pick_splits counts these tiles.
GEMM_TILE = {64: (128, 256), 32: (128, 128)}


def pick_splits(k_total: int, out_rows: int, out_cols: int, sms: int = 132, k_atom: int = 32) -> int:
    """split count for a wgrad GEMM, by a two-term cost model.  The persistent kernel runs ceil(tiles * splits / sms) waves
    of GEMM_TILE[k_atom] tiles (one CTA per SM), so the contraction costs flops / (peak * fill of the last wave) (to_qkv's
    fp16 wgrad, a 2304 x 768 output in 128 x 256 tiles: 54 tiles, 1 split = 0.41 waves, 2 splits = 0.82, 4 splits = 1.64);
    the partial sums cost one fp32 write and one read per split.  Each split contracts a multiple of one k-block (32 fp32 /
    64 fp16 elements) and at least 256 rows."""
    tm, tn = GEMM_TILE[k_atom]
    tiles = -(-out_rows // tm) * -(-out_cols // tn)
    peak = 0.99e15 if k_atom == 64 else 0.495e15       # H100 SXM dense f16 / tf32 tensor rates (data sheet)
    t_mma = 2.0 * k_total * out_rows * out_cols / peak
    best, best_t = 1, float("inf")
    s = 1
    while s <= 32 and k_total % (s * k_atom) == 0 and (s == 1 or k_total // s >= 256):
        work = tiles * s
        fill = work / (-(-work // sms) * sms)
        t = t_mma / fill + (8.0 * s * out_rows * out_cols / 6e12 if s > 1 else 0.0)
        if t < best_t * 0.98:                            # a larger count has to buy at least 2 %
            best, best_t = s, t
        s *= 2
    return best


# ------------------------------------------------------------------------ operand preparation
def split_tf32_lo(x: Tensor) -> Tensor:
    """x - trunc_tf32(x): the residue the 3xTF32 product feeds back in"""
    _req(x, "x")
    lo = torch.empty_like(x)
    _lib.check(_lib.lib().b200vq_split_tf32_lo(_p(x), _p(lo), x.numel(), _stream()), "split_tf32_lo")
    return lo


def to_half(x: Tensor, scale: Optional[Tensor] = None) -> Tensor:
    """fp16(x * scale), saturating; scale is a device scalar (element 0 of a grad_scale() pair) or None"""
    _req(x, "x"); _req(scale, "scale")
    out = torch.empty(x.shape, device=x.device, dtype=_HALF)
    _lib.check(_lib.lib().b200vq_to_half(_p(x), _p(out), x.numel(), _p(scale), _stream()), "to_half")
    return out


GRAD_TARGET_LOG2 = 6   # max|g| * S ~ 2^6: ~2^10 of headroom to fp16's 65504, full precision down to 2^-20 of max|g|


def grad_scale(g: Tensor, target_log2: int = GRAD_TARGET_LOG2) -> Tensor:
    """-> device tensor [S, 1/S], S the power of two that puts max|g| at ~2^target_log2 (no host sync)"""
    _req(g, "g")
    L = _lib.lib()
    ws_bytes = L.b200vq_grad_scale_workspace_bytes()
    ws = torch.empty(ws_bytes // 4, device=g.device, dtype=torch.float32)
    scale2 = torch.empty(2, device=g.device, dtype=torch.float32)
    _lib.check(L.b200vq_grad_scale(_p(g), g.numel(), int(target_log2), _p(scale2), _p(ws), ws_bytes, _stream()), "grad_scale")
    return scale2


# ------------------------------------------------------------------------------------- LayerNorm
def layernorm_fwd(x: Tensor, gamma: Tensor, beta: Tensor, round_out: bool, out_half: bool = False) -> Tuple[Tensor, Tensor, Tensor]:
    _req(x, "x"); _req(gamma, "gamma"); _req(beta, "beta")
    D = x.shape[-1]
    M = x.numel() // D
    y = torch.empty(x.shape, device=x.device, dtype=_HALF if out_half else torch.float32)
    mean = torch.empty(M, device=x.device, dtype=torch.float32)
    rstd = torch.empty(M, device=x.device, dtype=torch.float32)
    _lib.check(_lib.lib().b200vq_layernorm_fwd(_p(x), _p(gamma), _p(beta), None if out_half else _p(y), _p(y) if out_half else None,
                                               _p(mean), _p(rstd), M, D, int(round_out), _stream()), "layernorm_fwd")
    return y, mean, rstd


def layernorm_bwd(dy: Tensor, x: Tensor, mean: Tensor, rstd: Tensor, gamma: Tensor, dres: Optional[Tensor],
                  round_out: bool = False, want_colsum: bool = False, half_scale: Optional[Tensor] = None,
                  dy_scale: Optional[Tensor] = None):
    """-> (dx, dgamma, dbeta) or, with want_colsum, (dx, dgamma, dbeta, colsum(dx)); with half_scale (device
    scalar) a further element: the fp16 copy fp16(dx * scale).  dy may be fp16 (the scaled output of an fp16 dgrad
    GEMM): it is multiplied by the device scalar dy_scale (1/S) as it is read."""
    dy_half = dy.dtype == _HALF
    _req(dy, "dy", _HALF if dy_half else torch.float32); _req(x, "x"); _req(dres, "dres"); _req(half_scale, "half_scale")
    _req(dy_scale, "dy_scale")
    D = x.shape[-1]
    M = x.numel() // D
    L = _lib.lib()
    ws_bytes = L.b200vq_layernorm_bwd_workspace_bytes(D)
    ws = torch.empty(ws_bytes // 4, device=x.device, dtype=torch.float32)
    dx = torch.empty_like(x)
    dx16 = torch.empty(x.shape, device=x.device, dtype=_HALF) if half_scale is not None else None
    dgamma = torch.empty(D, device=x.device, dtype=torch.float32)
    dbeta = torch.empty(D, device=x.device, dtype=torch.float32)
    dxsum = torch.empty(D, device=x.device, dtype=torch.float32) if want_colsum else None
    _lib.check(L.b200vq_layernorm_bwd(_p(dy), int(dy_half), _p(dy_scale), _p(x), _p(mean), _p(rstd), _p(gamma), _p(dres), _p(dx), _p(dx16), _p(half_scale),
                                      _p(dgamma), _p(dbeta), _p(dxsum), M, D, int(round_out), _p(ws), ws_bytes, _stream()),
               "layernorm_bwd")
    res = (dx, dgamma, dbeta) + ((dxsum,) if want_colsum else ())
    return res + ((dx16,) if half_scale is not None else ())


# ------------------------------------------------------------------------------------- attention
def attention_fwd(qkv: Tensor, B: int, N: int, heads: int, dh: int, scale: float, round_out: bool,
                  out_half: bool = False) -> Tuple[Tensor, Tensor]:
    _req(qkv, "qkv")
    out = torch.empty(B * N, heads * dh, device=qkv.device, dtype=_HALF if out_half else torch.float32)
    lse = torch.empty(B * heads * N, device=qkv.device, dtype=torch.float32)
    _lib.check(_lib.lib().b200vq_attention_fwd(_p(qkv), _p(out), int(out_half), _p(lse), B, N, heads, dh, scale, int(round_out),
                                               _stream()), "attention_fwd")
    return out, lse


def attention_bwd(qkv: Tensor, out: Tensor, lse: Tensor, dout: Tensor, B: int, N: int, heads: int, dh: int,
                  scale: float, round_out: bool, half_scale: Optional[Tensor] = None) -> Tensor:
    """dqkv (fp32; or, with half_scale, fp16(dqkv * scale)).  `out` is the forward's output in whichever dtype it stored."""
    _req(qkv, "qkv"); _req(out, "out", out.dtype if out.dtype == _HALF else torch.float32); _req(lse, "lse"); _req(dout, "dout")
    _req(half_scale, "half_scale")
    dq_half = half_scale is not None
    dqkv = torch.empty(qkv.shape, device=qkv.device, dtype=_HALF if dq_half else torch.float32)
    delta = torch.empty_like(lse)
    _lib.check(_lib.lib().b200vq_attention_bwd(_p(qkv), _p(out), int(out.dtype == _HALF), _p(lse), _p(dout), _p(dqkv), int(dq_half),
                                               _p(half_scale), _p(delta), B, N, heads, dh, scale, int(round_out), _stream()),
               "attention_bwd")
    return dqkv


def attention_f16_fwd(qkv: Tensor, B: int, N: int, heads: int, dh: int, scale: float) -> Tuple[Tensor, Tensor]:
    """fp16-operand core (dh == 64): qkv fp16 -> (out fp16, lse fp32)"""
    _req(qkv, "qkv", _HALF)
    out = torch.empty(B * N, heads * dh, device=qkv.device, dtype=_HALF)
    lse = torch.empty(B * heads * N, device=qkv.device, dtype=torch.float32)
    _lib.check(_lib.lib().b200vq_attention_f16_fwd(_p(qkv), _p(out), _p(lse), B, N, heads, dh, scale, _stream()), "attention_f16_fwd")
    return out, lse


def attention_f16_bwd(qkv: Tensor, out: Tensor, lse: Tensor, dout: Tensor, B: int, N: int, heads: int, dh: int,
                      scale: float) -> Tensor:
    """dqkv fp16 from dout fp16 (dout may carry a power-of-two gradient scale; dqkv then carries the same one)"""
    _req(qkv, "qkv", _HALF); _req(out, "out", _HALF); _req(lse, "lse"); _req(dout, "dout", _HALF)
    dqkv = torch.empty_like(qkv)
    delta = torch.empty_like(lse)
    _lib.check(_lib.lib().b200vq_attention_f16_bwd(_p(qkv), _p(out), _p(lse), _p(dout), _p(dqkv), _p(delta), B, N, heads, dh, scale,
                                                   _stream()), "attention_f16_bwd")
    return dqkv


def attention_exact_fwd(qkv: Tensor, B: int, N: int, heads: int, dh: int, scale: float) -> Tuple[Tensor, Tensor]:
    _req(qkv, "qkv")
    out = torch.empty(B * N, heads * dh, device=qkv.device, dtype=torch.float32)
    lse = torch.empty(B * heads * N, device=qkv.device, dtype=torch.float32)
    _lib.check(_lib.lib().b200vq_attention_exact_fwd(_p(qkv), _p(out), _p(lse), B, N, heads, dh, scale, _stream()),
               "attention_exact_fwd")
    return out, lse


def attention_exact_bwd(qkv: Tensor, out: Tensor, lse: Tensor, dout: Tensor, B: int, N: int, heads: int, dh: int,
                        scale: float) -> Tensor:
    _req(qkv, "qkv"); _req(out, "out"); _req(lse, "lse"); _req(dout, "dout")
    dqkv = torch.empty_like(qkv)
    delta = torch.empty_like(lse)
    _lib.check(_lib.lib().b200vq_attention_exact_bwd(_p(qkv), _p(out), _p(lse), _p(dout), _p(dqkv), _p(delta), B, N, heads, dh,
                                                     scale, _stream()), "attention_exact_bwd")
    return dqkv


# ------------------------------------------------------------------------------------- quantiser
def vq_fwd(z: Tensor, E: Tensor, depth: int, beta: float, use_norm: bool = True) -> Tuple[Tensor, Tensor, Tensor]:
    """z [..., D], E [K, D] -> (straight-through value like z, loss scalar, idx int64 [M, depth]); D a multiple of 32
    from 32 to 256"""
    _req(z, "z"); _req(E, "embedding.weight")
    K, D = E.shape
    M = z.numel() // D
    L = _lib.lib()
    ws_bytes = L.b200vq_vq_fwd_workspace_bytes(M, K, D, depth)
    ws = torch.empty(ws_bytes // 4, device=z.device, dtype=torch.float32)
    out = torch.empty_like(z)
    idx = torch.empty(M, depth, device=z.device, dtype=torch.int64)
    loss = torch.empty((), device=z.device, dtype=torch.float32)
    _lib.check(L.b200vq_vq_fwd(_p(z), _p(E), _p(out), _p(idx), _p(loss), M, K, D, depth, float(beta), int(use_norm), _p(ws),
                               ws_bytes, _stream()), "vq_fwd")
    return out, loss, idx


def vq_bwd(z: Tensor, E: Tensor, idx: Tensor, g_out: Optional[Tensor], g_loss: Optional[Tensor], residual: bool,
           beta: float, use_norm: bool = True) -> Tuple[Tensor, Tensor]:
    _req(z, "z"); _req(E, "embedding.weight"); _req(idx, "idx", torch.int64); _req(g_out, "g_out"); _req(g_loss, "g_loss")
    K, D = E.shape
    M = z.numel() // D
    depth = idx.shape[-1] if idx.dim() == 2 else 1
    gz = torch.empty_like(z)
    gE = torch.empty_like(E)
    _lib.check(_lib.lib().b200vq_vq_bwd(_p(z), _p(E), _p(idx), _p(g_out), _p(g_loss), _p(gz), _p(gE), M, K, D, depth,
                                        int(residual), float(beta), int(use_norm), _stream()), "vq_bwd")
    return gz, gE


def vq_bwd_deterministic(z: Tensor, E: Tensor, idx: Tensor, g_out: Optional[Tensor], g_loss: Optional[Tensor], residual: bool,
                         beta: float, use_norm: bool = True) -> Tuple[Tensor, Tensor]:
    """vq_bwd with a bit-reproducible codebook gradient: gz is vq_bwd's bit for bit, gE is summed in an order that
    depends only on idx and the shape (no float atomics)"""
    _req(z, "z"); _req(E, "embedding.weight"); _req(idx, "idx", torch.int64); _req(g_out, "g_out"); _req(g_loss, "g_loss")
    K, D = E.shape
    M = z.numel() // D
    depth = idx.shape[-1] if idx.dim() == 2 else 1
    L = _lib.lib()
    ws_bytes = L.b200vq_vq_bwd_deterministic_workspace_bytes(M, K, D, depth)
    ws = torch.empty(max(ws_bytes, 1), device=z.device, dtype=torch.uint8)
    gz = torch.empty_like(z)
    gE = torch.empty_like(E)
    _lib.check(L.b200vq_vq_bwd_deterministic(_p(z), _p(E), _p(idx), _p(g_out), _p(g_loss), _p(gz), _p(gE), M, K, D, depth,
                                             int(residual), float(beta), int(use_norm), _p(ws), ws_bytes, _stream()),
               "vq_bwd_deterministic")
    return gz, gE


def vq_fwd_ema(z: Tensor, E: Tensor, depth: int, beta: float, use_norm: bool = True, stats: bool = True,
               deterministic: bool = False) -> Tuple[Tensor, Tensor, Tensor, Optional[Tensor]]:
    """EMA-codebook lookup: (out, loss, idx) as vq_fwd (the loss without its codebook term) and, with stats, one flat fp32
    buffer [K * (D + 1)]: the per-code sums s [K, D] followed by the counts n [K] -- the one tensor the replicas all-reduce.
    deterministic: s summed in a fixed order."""
    _req(z, "z"); _req(E, "embedding.weight")
    K, D = E.shape
    M = z.numel() // D
    L = _lib.lib()
    ws_bytes = L.b200vq_vq_fwd_ema_workspace_bytes(M, K, D, depth, int(deterministic))
    ws = torch.empty(max(ws_bytes, 1), device=z.device, dtype=torch.uint8)
    out = torch.empty_like(z)
    idx = torch.empty(M, depth, device=z.device, dtype=torch.int64)
    loss = torch.empty((), device=z.device, dtype=torch.float32)
    buf = torch.empty(K * (D + 1), device=z.device, dtype=torch.float32) if stats else None
    sums, counts = (buf[:K * D], buf[K * D:]) if stats else (None, None)
    _lib.check(L.b200vq_vq_fwd_ema(_p(z), _p(E), _p(out), _p(idx), _p(loss), _p(counts), _p(sums), M, K, D, depth, float(beta),
                                   int(use_norm), int(deterministic), _p(ws), ws_bytes, _stream()), "vq_fwd_ema")
    return out, loss, idx, buf


def vq_ema_update(stats: Tensor, cluster_size: Tensor, embed_avg: Tensor, weight: Tensor, decay: float, eps: float) -> None:
    """in place: the EMA update of cluster_size [K], embed_avg [K, D] and weight [K, D] from vq_fwd_ema's flat statistics"""
    _req(stats, "stats"); _req(cluster_size, "cluster_size"); _req(embed_avg, "embed_avg"); _req(weight, "embedding.weight")
    K, D = weight.shape
    if stats.numel() != K * (D + 1) or cluster_size.numel() != K or embed_avg.shape != weight.shape:
        raise RuntimeError(f"b200vq: vq_ema_update shapes: stats {tuple(stats.shape)}, cluster_size {tuple(cluster_size.shape)}, "
                           f"embed_avg {tuple(embed_avg.shape)}, weight {tuple(weight.shape)}")
    _lib.check(_lib.lib().b200vq_vq_ema_update(_p(stats[K * D:]), _p(stats), _p(cluster_size), _p(embed_avg), _p(weight), K, D,
                                               float(decay), float(eps), _stream()), "vq_ema_update")


def vq_embed(E: Tensor, codes: Tensor, depth: int, use_norm: bool = True) -> Tensor:
    _req(E, "embedding.weight"); _req(codes, "codes", torch.int64)
    K, D = E.shape
    M = codes.numel() // depth
    out = torch.empty(M, D, device=E.device, dtype=torch.float32)
    _lib.check(_lib.lib().b200vq_vq_embed(_p(E), _p(codes), _p(out), M, K, D, depth, int(use_norm), _stream()), "vq_embed")
    return out


# ---------------------------------------------------------------------------- layout / reductions
def _pair(p):
    return (int(p[0]), int(p[1])) if isinstance(p, (tuple, list)) else (int(p), int(p))


def patchify(img: Tensor, p, round_out: bool) -> Tensor:
    """p: patch side or (height, width)"""
    _req(img, "img")
    B, C, H, W = img.shape
    ph, pw = _pair(p)
    out = torch.empty(B * (H // ph) * (W // pw), C * ph * pw, device=img.device, dtype=torch.float32)
    _lib.check(_lib.lib().b200vq_patchify(_p(img), _p(out), B, C, H, W, ph, pw, int(round_out), _stream()), "patchify")
    return out


def unpatchify(tok: Tensor, bias: Optional[Tensor], B: int, C: int, H: int, W: int, p) -> Tensor:
    _req(tok, "tok"); _req(bias, "bias")
    ph, pw = _pair(p)
    img = torch.empty(B, C, H, W, device=tok.device, dtype=torch.float32)
    _lib.check(_lib.lib().b200vq_unpatchify(_p(tok), _p(bias), _p(img), B, C, H, W, ph, pw, _stream()), "unpatchify")
    return img


def colsum(x: Tensor) -> Tensor:
    _req(x, "x")
    N = x.shape[-1]
    M = x.numel() // N
    L = _lib.lib()
    ws_bytes = L.b200vq_colsum_workspace_bytes(N)
    ws = torch.empty(ws_bytes // 4, device=x.device, dtype=torch.float32)
    out = torch.empty(N, device=x.device, dtype=torch.float32)
    _lib.check(L.b200vq_colsum(_p(x), N, M, N, _p(out), _p(ws), ws_bytes, _stream()), "colsum")
    return out


def round_tf32(x: Tensor, out: Optional[Tensor] = None) -> Tensor:
    _req(x, "x")
    if out is None:
        out = torch.empty_like(x)
    _lib.check(_lib.lib().b200vq_round_tf32(_p(x), _p(out), x.numel(), _stream()), "round_tf32")
    return out


def add_rows_mod(x: Tensor, table: Tensor) -> Tensor:
    """x [M, D] + table[m % R] (R = table rows)"""
    _req(x, "x"); _req(table, "table")
    D = x.shape[-1]
    M = x.numel() // D
    R = table.numel() // D
    out = torch.empty_like(x)
    _lib.check(_lib.lib().b200vq_add_rows_mod(_p(x), _p(table), _p(out), M, D, R, _stream()), "add_rows_mod")
    return out


# ------------------------------------------------------------------- stage-2 transformer (SURVEY.md 8f-3)
def attention_causal_fwd(qkv: Tensor, B: int, N: int, heads: int, dh: int, scale: float, cond_len: int, exact: bool,
                         round_out: bool = False) -> Tuple[Tensor, Tensor]:
    """masked attention core of the stage-2 blocks: query q sees key k iff k <= max(q, cond_len - 1)"""
    _req(qkv, "qkv")
    out = torch.empty(B * N, heads * dh, device=qkv.device, dtype=torch.float32)
    lse = torch.empty(B * heads * N, device=qkv.device, dtype=torch.float32)
    _lib.check(_lib.lib().b200vq_attention_causal_fwd(_p(qkv), _p(out), _p(lse), B, N, heads, dh, scale, int(cond_len), int(exact),
                                                      int(round_out), _stream()), "attention_causal_fwd")
    return out, lse


def attention_causal_bwd(qkv: Tensor, out: Tensor, lse: Tensor, dout: Tensor, B: int, N: int, heads: int, dh: int, scale: float,
                         cond_len: int, exact: bool, round_out: bool = False) -> Tensor:
    _req(qkv, "qkv"); _req(out, "out"); _req(lse, "lse"); _req(dout, "dout")
    dqkv = torch.empty_like(qkv)
    delta = torch.empty_like(lse)
    _lib.check(_lib.lib().b200vq_attention_causal_bwd(_p(qkv), _p(out), _p(lse), _p(dout), _p(dqkv), _p(delta), B, N, heads, dh, scale,
                                                      int(cond_len), int(exact), int(round_out), _stream()), "attention_causal_bwd")
    return dqkv


def time_mix_fwd(x: Tensor, w: Tensor, T: int, round_out: bool = False) -> Tensor:
    """x [M = B*T, C], w [C] -> x * w + shift(x) * (1 - w)"""
    _req(x, "x"); _req(w, "time_mix")
    M, C = x.shape
    y = torch.empty_like(x)
    _lib.check(_lib.lib().b200vq_time_mix_fwd(_p(x), _p(w), _p(y), M, T, C, int(round_out), _stream()), "time_mix_fwd")
    return y


def time_mix_bwd(g: Tensor, x: Tensor, w: Tensor, T: int) -> Tuple[Tensor, Tensor]:
    """-> (gx, gw)"""
    _req(g, "g"); _req(x, "x"); _req(w, "time_mix")
    M, C = x.shape
    L = _lib.lib()
    part = torch.empty(L.b200vq_time_mix_bwd_workspace_bytes(M, C) // (4 * C), C, device=x.device, dtype=torch.float32)
    gx = torch.empty_like(x)
    _lib.check(L.b200vq_time_mix_bwd(_p(g), _p(x), _p(w), _p(gx), _p(part), M, T, C, _stream()), "time_mix_bwd")
    return gx, colsum(part)


def sqrelu(x: Tensor, g: Optional[Tensor] = None, round_out: bool = False) -> Tensor:
    """g is None: relu(x)^2; otherwise g * 2 relu(x) (x the pre-activation)"""
    _req(x, "x"); _req(g, "g")
    y = torch.empty_like(x)
    _lib.check(_lib.lib().b200vq_sqrelu(_p(x), _p(g), _p(y), x.numel(), int(g is not None), int(round_out), _stream()), "sqrelu")
    return y


def token_embed_fwd(conds: Tensor, codes: Tensor, Wc: Tensor, pos_c: Tensor, Wi: Tensor, pos_i: Tensor) -> Tensor:
    """conds int64 [B, Tc], codes int64 [B, Ti] -> x [B * (Tc + Ti), C]"""
    _req(conds, "conds", torch.int64); _req(codes, "codes", torch.int64)
    _req(Wc, "tok_emb_cond.weight"); _req(pos_c, "pos_emb_cond"); _req(Wi, "tok_emb_code.weight"); _req(pos_i, "pos_emb_code")
    B, Tc = conds.shape
    Ti = codes.shape[1]
    C = Wi.shape[1]
    x = torch.empty(B * (Tc + Ti), C, device=Wi.device, dtype=torch.float32)
    _lib.check(_lib.lib().b200vq_token_embed_fwd(_p(conds), _p(codes), _p(Wc), _p(pos_c), _p(Wi), _p(pos_i), _p(x), B, Tc, Ti, C,
                                                 Wc.shape[0], Wi.shape[0], _stream()), "token_embed_fwd")
    return x


def token_embed_bwd(conds: Tensor, codes: Tensor, g: Tensor, Vc: int, Vi: int) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
    """-> (gWc [Vc, C], gpos_c [Tc, C], gWi [Vi, C], gpos_i [Ti, C])"""
    _req(conds, "conds", torch.int64); _req(codes, "codes", torch.int64); _req(g, "g")
    B, Tc = conds.shape
    Ti = codes.shape[1]
    C = g.shape[-1]
    gWc = torch.empty(Vc, C, device=g.device, dtype=torch.float32)
    gWi = torch.empty(Vi, C, device=g.device, dtype=torch.float32)
    gpc = torch.empty(Tc, C, device=g.device, dtype=torch.float32)
    gpi = torch.empty(Ti, C, device=g.device, dtype=torch.float32)
    _lib.check(_lib.lib().b200vq_token_embed_bwd(_p(conds), _p(codes), _p(g), _p(gWc), _p(gpc), _p(gWi), _p(gpi), B, Tc, Ti, C, Vc, Vi,
                                                 _stream()), "token_embed_bwd")
    return gWc, gpc, gWi, gpi


def token_embed_bwd_deterministic(conds: Tensor, codes: Tensor, g: Tensor, Vc: int, Vi: int) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
    """token_embed_bwd with gWc / gWi summed in an order that depends only on the ids and the shape (no float atomics);
    gpos_c / gpos_i are token_embed_bwd's bit for bit"""
    _req(conds, "conds", torch.int64); _req(codes, "codes", torch.int64); _req(g, "g")
    B, Tc = conds.shape
    Ti = codes.shape[1]
    C = g.shape[-1]
    L = _lib.lib()
    ws_bytes = L.b200vq_token_embed_bwd_deterministic_workspace_bytes(B, Tc, Ti, C, Vc, Vi)
    ws = torch.empty(max(ws_bytes, 1), device=g.device, dtype=torch.uint8)
    gWc = torch.empty(Vc, C, device=g.device, dtype=torch.float32)
    gWi = torch.empty(Vi, C, device=g.device, dtype=torch.float32)
    gpc = torch.empty(Tc, C, device=g.device, dtype=torch.float32)
    gpi = torch.empty(Ti, C, device=g.device, dtype=torch.float32)
    _lib.check(L.b200vq_token_embed_bwd_deterministic(_p(conds), _p(codes), _p(g), _p(gWc), _p(gpc), _p(gWi), _p(gpi), B, Tc, Ti, C,
                                                      Vc, Vi, _p(ws), ws_bytes, _stream()), "token_embed_bwd_deterministic")
    return gWc, gpc, gWi, gpi


def copy_rows(src: Tensor, B: int, T_src: int, T_dst: int, off_src: int, off_dst: int, n: int) -> Tensor:
    """src [B*T_src, C] -> dst [B*T_dst, C]: rows [off_dst, off_dst + n) of every batch entry copied from
    [off_src, off_src + n), the rest zero"""
    _req(src, "src")
    C = src.shape[-1]
    dst = torch.empty(B * T_dst, C, device=src.device, dtype=torch.float32)
    _lib.check(_lib.lib().b200vq_copy_rows(_p(src), _p(dst), B, T_src, T_dst, off_src, off_dst, n, C, _stream()), "copy_rows")
    return dst


def decode_attention(qkv: Tensor, cache_k: Tensor, cache_v: Tensor, heads: int, hs: int, pos: int, scale: float) -> Tensor:
    """one sampling step: qkv [B, 3*C]; caches [B, Tmax, C] (row `pos` is written); -> out [B, C]"""
    _req(qkv, "qkv"); _req(cache_k, "cache_k"); _req(cache_v, "cache_v")
    B = qkv.shape[0]
    out = torch.empty(B, heads * hs, device=qkv.device, dtype=torch.float32)
    _lib.check(_lib.lib().b200vq_decode_attention(_p(qkv), _p(cache_k), _p(cache_v), _p(out), B, heads, hs, cache_k.shape[1], int(pos),
                                                  scale, _stream()), "decode_attention")
    return out


# ----------------------------------------------------------------- stage-2 RQTransformer (reference layers.py:306-547)
def short_attention_fwd(qkv: Tensor, nseq: int, D: int, heads: int, hs: int, scale: float, cond_len: int = 0) -> Tensor:
    """causal attention over nseq independent sequences of D <= 16 tokens: qkv [nseq*D, 3C] -> out [nseq*D, C] (fp32 FMA)"""
    _req(qkv, "qkv")
    out = torch.empty(nseq * D, heads * hs, device=qkv.device, dtype=torch.float32)
    _lib.check(_lib.lib().b200vq_short_attention_fwd(_p(qkv), _p(out), nseq, D, heads, hs, int(cond_len), scale, _stream()),
               "short_attention_fwd")
    return out


def short_attention_bwd(qkv: Tensor, dout: Tensor, nseq: int, D: int, heads: int, hs: int, scale: float, cond_len: int = 0) -> Tensor:
    """dqkv [nseq*D, 3C], the scores recomputed from qkv"""
    _req(qkv, "qkv"); _req(dout, "dout")
    dqkv = torch.empty_like(qkv)
    _lib.check(_lib.lib().b200vq_short_attention_bwd(_p(qkv), _p(dout), _p(dqkv), nseq, D, heads, hs, int(cond_len), scale, _stream()),
               "short_attention_bwd")
    return dqkv


def rq_embed_fwd(conds: Tensor, codes: Tensor, Wc: Tensor, pos_c: Tensor, Wi: Tensor, pos_i: Tensor) -> Tensor:
    """conds int64 [B, Tc], codes int64 [B, T, D] -> x [B * (Tc + T), C]: cond rows Wc[conds] + pos_c, code rows
    cumsum_C(Wi[codes[..., D-1]]) + pos_i"""
    _req(conds, "conds", torch.int64); _req(codes, "codes", torch.int64)
    _req(Wc, "tok_emb_cond.weight"); _req(pos_c, "pos_emb_cond"); _req(Wi, "tok_emb_code.weight"); _req(pos_i, "pos_emb_code")
    B, Tc = conds.shape
    _, T, D = codes.shape
    C = Wi.shape[1]
    x = torch.empty(B * (Tc + T), C, device=Wi.device, dtype=torch.float32)
    _lib.check(_lib.lib().b200vq_rq_embed_fwd(_p(conds), _p(codes), _p(Wc), _p(pos_c), _p(Wi), _p(pos_i), _p(x), B, Tc, T, D, C,
                                              Wc.shape[0], Wi.shape[0], _stream()), "rq_embed_fwd")
    return x


def rq_embed_bwd(conds: Tensor, codes: Tensor, g: Tensor, Vc: int, Vi: int,
                 deterministic: bool = False) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
    """-> (gWc [Vc, C], gpos_c [Tc, C], gWi [Vi, C], gpos_i [T, C]); deterministic: gWc / gWi summed in a fixed order"""
    _req(conds, "conds", torch.int64); _req(codes, "codes", torch.int64); _req(g, "g")
    B, Tc = conds.shape
    _, T, D = codes.shape
    C = g.shape[-1]
    gWc = torch.empty(Vc, C, device=g.device, dtype=torch.float32)
    gWi = torch.empty(Vi, C, device=g.device, dtype=torch.float32)
    gpc = torch.empty(Tc, C, device=g.device, dtype=torch.float32)
    gpi = torch.empty(T, C, device=g.device, dtype=torch.float32)
    L = _lib.lib()
    args = (_p(conds), _p(codes), _p(g), _p(gWc), _p(gpc), _p(gWi), _p(gpi), B, Tc, T, D, C, Vc, Vi)
    if deterministic:
        ws_bytes = L.b200vq_rq_embed_bwd_deterministic_workspace_bytes(B, Tc, T, D, C, Vc, Vi)
        ws = torch.empty(max(ws_bytes, 1), device=g.device, dtype=torch.uint8)
        _lib.check(L.b200vq_rq_embed_bwd_deterministic(*args, _p(ws), ws_bytes, _stream()), "rq_embed_bwd_deterministic")
    else:
        _lib.check(L.b200vq_rq_embed_bwd(*args, _stream()), "rq_embed_bwd")
    return gWc, gpc, gWi, gpi


def rq_depth_input_fwd(h: Tensor, codes: Tensor, Wi: Tensor, pos_d: Tensor) -> Tensor:
    """h [B*T, C], codes int64 [B, T, D], pos_d [D-1, C] -> v [B*T*D, C]: v[s, 0] = h[s], v[s, d] = cumsum_C(Wi[codes[s, d-1]]) +
    pos_d[d-1]"""
    _req(h, "h"); _req(codes, "codes", torch.int64); _req(Wi, "tok_emb_code.weight"); _req(pos_d, "pos_emb_depth")
    D = codes.shape[-1]
    nseq = codes.numel() // D
    C = Wi.shape[1]
    v = torch.empty(nseq * D, C, device=h.device, dtype=torch.float32)
    _lib.check(_lib.lib().b200vq_rq_depth_input_fwd(_p(h), _p(codes), _p(Wi), _p(pos_d), _p(v), nseq, D, C, Wi.shape[0], _stream()),
               "rq_depth_input_fwd")
    return v


def rq_depth_input_bwd(codes: Tensor, g: Tensor, Vi: int, deterministic: bool = False) -> Tuple[Tensor, Tensor, Tensor]:
    """-> (gh [B*T, C], gWi [Vi, C], gpos_d [D-1, C]); deterministic: gWi summed in a fixed order"""
    _req(codes, "codes", torch.int64); _req(g, "g")
    D = codes.shape[-1]
    nseq = codes.numel() // D
    C = g.shape[-1]
    gh = torch.empty(nseq, C, device=g.device, dtype=torch.float32)
    gWi = torch.empty(Vi, C, device=g.device, dtype=torch.float32)
    gpd = torch.empty(D - 1, C, device=g.device, dtype=torch.float32)
    L = _lib.lib()
    args = (_p(codes), _p(g), _p(gh), _p(gWi), _p(gpd), nseq, D, C, Vi)
    if deterministic:
        ws_bytes = L.b200vq_rq_depth_input_bwd_deterministic_workspace_bytes(nseq, D, C, Vi)
        ws = torch.empty(max(ws_bytes, 1), device=g.device, dtype=torch.uint8)
        _lib.check(L.b200vq_rq_depth_input_bwd_deterministic(*args, _p(ws), ws_bytes, _stream()), "rq_depth_input_bwd_deterministic")
    else:
        _lib.check(L.b200vq_rq_depth_input_bwd(*args, _stream()), "rq_depth_input_bwd")
    return gh, gWi, gpd


def code_sum_embed(codes: Tensor, n: int, Wi: Tensor, pos: Tensor) -> Tensor:
    """codes int64 [B, >= n] (rows may be strided; each row's first n entries are read) -> out [B, C] =
    sum_{j < n} Wi[codes[b, j]] + pos (one [C] row)"""
    _req(Wi, "tok_emb_code.weight"); _req(pos, "pos")
    if not codes.is_cuda or codes.dtype != torch.int64 or codes.stride(1) != 1:
        raise RuntimeError("b200vq: `codes` must be a CUDA int64 matrix with unit column stride")
    B = codes.shape[0]
    C = Wi.shape[1]
    out = torch.empty(B, C, device=Wi.device, dtype=torch.float32)
    _lib.check(_lib.lib().b200vq_code_sum_embed(_p(codes), codes.stride(0), int(n), _p(Wi), _p(pos), _p(out), B, C, Wi.shape[0], _stream()),
               "code_sum_embed")
    return out
