"""CPU oracle for the ViT-VQGAN hot path -- TEST INFRASTRUCTURE ONLY.

This file restates, as pure functions over a flat ``state_dict``, the algorithm of the
reference's ``enhancing/modules/stage1/layers.py`` (ViTEncoder / ViTDecoder) and
``enhancing/modules/stage1/quantizers.py`` (VectorQuantizer incl. residual mode), plus the two
``nn.Linear`` layers the reference's ``ViTVQ`` LightningModule puts between them
(``vitvqgan.py:38-39,63,69``).  It exists so that ``tests/``, ``__graft_entry__.smoke()`` and
``bench.py``'s ``cpu_baseline`` / ``--impl reference`` legs have something to check the CUDA path
against on a machine without a reference checkout.  Nothing under the product
package (``enhancing_transformers_b200/``) may import it.

Parity pin: the reference ships no tests and no golden vectors (SURVEY.md section 4), so this
oracle is pinned against outputs of the *reference itself*, generated from a reference checkout by
``oracle/gen_golden.py`` (which imports the reference modules from a reference checkout by file
path) and committed under ``tests/golden/``.  ``tests/test_oracle_golden.py`` replays them.

Arithmetic: fp32 torch CPU ops (the reference's own arithmetic lives in ATen, SURVEY.md
section 8c); gradients come from autograd over these functions, except for the quantiser, whose
backward is additionally written out by hand in numpy (``vq_backward_np``) because the CUDA
kernels implement exactly those closed forms.
"""
from __future__ import annotations

import math
from typing import Dict, Optional, Tuple

import numpy as np
import torch

Tensor = torch.Tensor
LN_EPS = 1e-5          # nn.LayerNorm default, reference layers.py:88,143
NORM_EPS = 1e-12       # F.normalize default, reference quantizers.py:24


# ----------------------------------------------------------------------------------------------
# positional table (reference layers.py:21-68)
# ----------------------------------------------------------------------------------------------
def _sincos_1d(half_dim: int, pos: np.ndarray) -> np.ndarray:
    """layers.py:49-68: omega_j = 10000^(-j/(half_dim/2)), float64; [sin | cos] halves."""
    assert half_dim % 2 == 0
    j = np.arange(half_dim // 2, dtype=np.float64)
    omega = 1.0 / 10000.0 ** (j / (half_dim / 2.0))
    ang = pos.reshape(-1).astype(np.float64)[:, None] * omega[None, :]
    return np.concatenate([np.sin(ang), np.cos(ang)], axis=1)


def sincos_pos_embed(dim: int, grid_hw: Tuple[int, int]) -> np.ndarray:
    """layers.py:21-46.  The reference calls ``np.meshgrid(grid_w, grid_h)`` ("w goes first",
    :30) so ``grid[0]`` varies along the width; the first half of the channels encodes that
    coordinate and the second half the row coordinate.  Returns float32 [gh*gw, dim]."""
    gh, gw = grid_hw
    ys, xs = np.arange(gh, dtype=np.float32), np.arange(gw, dtype=np.float32)
    col = np.broadcast_to(xs[None, :], (gh, gw))      # == meshgrid(grid_w, grid_h)[0]
    row = np.broadcast_to(ys[:, None], (gh, gw))      # == meshgrid(grid_w, grid_h)[1]
    first = _sincos_1d(dim // 2, col)
    second = _sincos_1d(dim // 2, row)
    return np.concatenate([first, second], axis=1).astype(np.float32)


# ----------------------------------------------------------------------------------------------
# transformer blocks (reference layers.py:85-150)
# ----------------------------------------------------------------------------------------------
def layer_norm(x: Tensor, w: Tensor, b: Tensor) -> Tensor:
    """PreNorm's nn.LayerNorm(dim): layers.py:88,92 (biased variance, eps inside sqrt)."""
    mu = x.mean(dim=-1, keepdim=True)
    var = ((x - mu) ** 2).mean(dim=-1, keepdim=True)
    return (x - mu) * torch.rsqrt(var + LN_EPS) * w + b


def attention(x: Tensor, w_qkv: Tensor, w_out: Tensor, b_out: Tensor, heads: int) -> Tensor:
    """layers.py:122-132.  to_qkv has no bias (:118); scale = dim_head**-0.5 applied to the
    scores after the product (:126); plain softmax, no mask (:127)."""
    B, N, _ = x.shape
    inner = w_qkv.shape[0] // 3
    dh = inner // heads
    qkv = x @ w_qkv.t()
    q, k, v = (t.reshape(B, N, heads, dh).permute(0, 2, 1, 3) for t in qkv.split(inner, dim=-1))
    s = (q @ k.transpose(-1, -2)) * (dh ** -0.5)
    p = torch.softmax(s, dim=-1)
    o = (p @ v).permute(0, 2, 1, 3).reshape(B, N, inner)
    return o @ w_out.t() + b_out


def feed_forward(x: Tensor, w1: Tensor, b1: Tensor, w2: Tensor, b2: Tensor) -> Tensor:
    """layers.py:98-105: Linear -> Tanh -> Linear."""
    return torch.tanh(x @ w1.t() + b1) @ w2.t() + b2


def transformer(x: Tensor, sd: Dict[str, Tensor], prefix: str, depth: int, heads: int) -> Tensor:
    """layers.py:145-150: x = attn(LN(x)) + x; x = ff(LN(x)) + x; final LayerNorm."""
    for i in range(depth):
        a, f = f"{prefix}layers.{i}.0.", f"{prefix}layers.{i}.1."
        x = attention(layer_norm(x, sd[a + "norm.weight"], sd[a + "norm.bias"]),
                      sd[a + "fn.to_qkv.weight"], sd[a + "fn.to_out.weight"], sd[a + "fn.to_out.bias"],
                      heads) + x
        x = feed_forward(layer_norm(x, sd[f + "norm.weight"], sd[f + "norm.bias"]),
                         sd[f + "fn.net.0.weight"], sd[f + "fn.net.0.bias"],
                         sd[f + "fn.net.2.weight"], sd[f + "fn.net.2.bias"]) + x
    return layer_norm(x, sd[prefix + "norm.weight"], sd[prefix + "norm.bias"])


def patchify(img: Tensor, p: int) -> Tensor:
    """[B,C,H,W] -> [B, (H/p)(W/p), C*p*p], patch vector ordered (c, ph, pw): the im2col view of
    Conv2d(kernel=stride=p) followed by 'b c h w -> b (h w) c' (layers.py:168-171)."""
    B, C, H, W = img.shape
    t = img.reshape(B, C, H // p, p, W // p, p).permute(0, 2, 4, 1, 3, 5)
    return t.reshape(B, (H // p) * (W // p), C * p * p)


def unpatchify(tok: Tensor, p: int, gh: int, gw: int, C: int) -> Tensor:
    """inverse of patchify: the pixel-shuffle store of ConvTranspose2d(kernel=stride=p)."""
    B = tok.shape[0]
    t = tok.reshape(B, gh, gw, C, p, p).permute(0, 3, 1, 4, 2, 5)
    return t.reshape(B, C, gh * p, gw * p)


def vit_encoder(sd: Dict[str, Tensor], img: Tensor, *, patch: int, depth: int, heads: int,
                prefix: str = "") -> Tensor:
    """ViTEncoder.forward, layers.py:177-182.  Conv2d weight [D,C,p,p] is a [D, C*p*p] GEMM."""
    w = sd[prefix + "to_patch_embedding.0.weight"]
    x = patchify(img, patch) @ w.reshape(w.shape[0], -1).t() + sd[prefix + "to_patch_embedding.0.bias"]
    x = x + sd[prefix + "en_pos_embedding"]
    return transformer(x, sd, prefix + "transformer.", depth, heads)


def vit_decoder(sd: Dict[str, Tensor], tok: Tensor, *, patch: int, depth: int, heads: int,
                grid_hw: Tuple[int, int], prefix: str = "") -> Tensor:
    """ViTDecoder.forward, layers.py:209-214.  ConvTranspose2d weight [D,C,p,p] is a
    [D, C*p*p] matrix applied on the right; bias is per output channel c (:204)."""
    x = tok + sd[prefix + "de_pos_embedding"]
    x = transformer(x, sd, prefix + "transformer.", depth, heads)
    w = sd[prefix + "to_pixel.1.weight"]
    C = w.shape[1]
    y = x @ w.reshape(w.shape[0], -1)
    y = y + sd[prefix + "to_pixel.1.bias"].repeat_interleave(patch * patch)
    return unpatchify(y, patch, grid_hw[0], grid_hw[1], C)


# ----------------------------------------------------------------------------------------------
# quantiser (reference quantizers.py:19-92)
# ----------------------------------------------------------------------------------------------
def l2norm(x: Tensor) -> Tensor:
    """BaseQuantizer.norm, quantizers.py:24: x / max(||x||_2, 1e-12) along the last dim."""
    return x / x.norm(dim=-1, keepdim=True).clamp_min(NORM_EPS)


def vq_distances(zn: Tensor, en: Tensor) -> Tensor:
    """quantizers.py:78-80, in the reference's association: (|z|^2 + |e|^2) - 2 * (z . e)."""
    return (zn ** 2).sum(dim=1, keepdim=True) + (en ** 2).sum(dim=1) - 2 * (zn @ en.t())


def vq_quantize(z: Tensor, E: Tensor, beta: float) -> Tuple[Tensor, Tensor, Tensor]:
    """VectorQuantizer.quantize, quantizers.py:74-92 (use_norm=True).  Returns the *normalised*
    selected code, the loss, and int64 indices shaped like z.shape[:-1]; argmin = first min."""
    D = E.shape[1]
    zf = z.reshape(-1, D)
    idx = torch.argmin(vq_distances(l2norm(zf), l2norm(E)), dim=1).reshape(z.shape[:-1])
    zq_n, z_n = l2norm(E[idx]), l2norm(z)
    loss = beta * ((zq_n.detach() - z_n) ** 2).mean() + ((zq_n - z_n.detach()) ** 2).mean()
    return zq_n, loss, idx


def vq_forward(z: Tensor, E: Tensor, beta: float = 0.25, use_residual: bool = False,
               num_quantizers: Optional[int] = None) -> Tuple[Tensor, Tensor, Tensor]:
    """BaseQuantizer.forward, quantizers.py:38-63 with straight_through=True (:69).

    Residual mode (:42-57): the residual starts as a *detached* copy of z, every depth
    re-normalises it, subtracts the unit-norm code (keeping that code's graph) and the
    per-depth losses are averaged; indices stack on a new last axis."""
    if not use_residual:
        zq, loss, idx = vq_quantize(z, E, beta)
    else:
        zq = torch.zeros_like(z)
        r = z.detach().clone()
        losses, idxs = [], []
        for _ in range(int(num_quantizers)):
            q, l, i = vq_quantize(r, E, beta)
            r = r - q
            zq = zq + q
            losses.append(l)
            idxs.append(i)
        loss = torch.stack(losses, dim=-1).mean()
        idx = torch.stack(idxs, dim=-1)
    out = z + (zq - z).detach()          # :60-61, value differs from zq in the last ulp
    return out, loss, idx


def decode_codes_embed(code: Tensor, E: Tensor, use_residual: bool) -> Tensor:
    """ViTVQ.decode_codes, vitvqgan.py:81-86: embedding -> norm -> (sum over depth)."""
    q = l2norm(E[code])
    return q.sum(-2) if use_residual else q


# --- explicit numpy restatement of the quantiser forward/backward (closed forms) --------------
def _np_norm(x: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    n = np.maximum(np.sqrt((x * x).sum(-1, keepdims=True, dtype=np.float32)), np.float32(NORM_EPS))
    return (x / n).astype(np.float32), n.astype(np.float32)


def vq_lookup_np(z: np.ndarray, E: np.ndarray) -> np.ndarray:
    """distance + argmin only (quantizers.py:75-83) in fp32 numpy; z [M,D], E [K,D] -> int64 [M]."""
    zn, _ = _np_norm(z.astype(np.float32))
    en, _ = _np_norm(E.astype(np.float32))
    d = ((zn * zn).sum(1, keepdims=True, dtype=np.float32) + (en * en).sum(1, dtype=np.float32)) \
        - np.float32(2) * (zn @ en.T)
    return d.argmin(axis=1).astype(np.int64)


def vq_top2_gap_f64(z: np.ndarray, E: np.ndarray) -> np.ndarray:
    """float64 gap between the best and second-best distance per row; rows with a gap below
    ~1e-6 are fp32 near-ties where any two correct implementations may disagree
    (SURVEY.md section 7 'Hard parts')."""
    z64, e64 = z.astype(np.float64), E.astype(np.float64)
    zn = z64 / np.maximum(np.linalg.norm(z64, axis=1, keepdims=True), NORM_EPS)
    en = e64 / np.maximum(np.linalg.norm(e64, axis=1, keepdims=True), NORM_EPS)
    d = (zn * zn).sum(1, keepdims=True) + (en * en).sum(1) - 2 * zn @ en.T
    part = np.partition(d, 1, axis=1)
    return part[:, 1] - part[:, 0]


def _np_norm_jt(x: np.ndarray, v: np.ndarray) -> np.ndarray:
    """J_n(x)^T v for n(x) = x / max(|x|, eps):  (v - xh (xh . v)) / |x|."""
    xh, n = _np_norm(x)
    return ((v - xh * (xh * v).sum(-1, keepdims=True)) / n).astype(np.float32)


def vq_backward_np(z: np.ndarray, E: np.ndarray, idx: np.ndarray, g_out: np.ndarray, g_loss: float,
                   beta: float = 0.25, use_residual: bool = False) -> Tuple[np.ndarray, np.ndarray]:
    """Closed-form gradients of (out, loss) = vq_forward(z, E) w.r.t. z and E, given upstream
    g_out (same shape as z) and scalar g_loss.  Mirrors what autograd derives from
    quantizers.py:38-63,85-92 (SURVEY.md section 8a rows Q3-Q5):

    * the straight-through output passes g_out to z unchanged and nothing to E;
    * plain mode:  dz += g_loss*beta*c*Jn(z)^T(zn - qn),  dE[idx] += g_loss*c*Jn(e)^T(qn - zn),
      c = 2/(M*D);
    * residual mode (T depths, loss = mean_t): z gets no loss gradient (the residual is a
      detached clone, :43); the code at depth s receives its own codebook term plus, through
      r_t = r_0 - sum_{s<t} q_s, minus the commitment gradient of every later depth.
    """
    D = E.shape[1]
    zf = z.reshape(-1, D).astype(np.float32)
    M = zf.shape[0]
    gz = g_out.reshape(-1, D).astype(np.float32).copy()
    gE = np.zeros_like(E, dtype=np.float32)
    c = np.float32(2.0 / (M * D))
    if not use_residual:
        ii = idx.reshape(-1)
        e = E[ii]
        qn, _ = _np_norm(e)
        zn, _ = _np_norm(zf)
        gz += np.float32(g_loss * beta) * c * _np_norm_jt(zf, zn - qn)
        np.add.at(gE, ii, np.float32(g_loss) * c * _np_norm_jt(e, qn - zn))
    else:
        T = idx.shape[-1]
        ii = idx.reshape(-1, T)
        gl = np.float32(g_loss / T)
        r = zf.copy()
        g_q = []            # gradient w.r.t. the normalised code emitted at each depth
        g_r = []            # commitment gradient w.r.t. the residual entering each depth
        for t in range(T):
            e = E[ii[:, t]]
            qn, _ = _np_norm(e)
            rn, _ = _np_norm(r)
            g_q.append(gl * c * (qn - rn))
            g_r.append(gl * np.float32(beta) * c * _np_norm_jt(r, rn - qn))
            r = r - qn
        for s in range(T):
            tot = g_q[s].copy()
            for t in range(s + 1, T):
                tot -= g_r[t]
            np.add.at(gE, ii[:, s], _np_norm_jt(E[ii[:, s]], tot))
    return gz.reshape(z.shape), gE


# ----------------------------------------------------------------------------------------------
# the unit of work bench.py measures (SURVEY.md section 8d)
# ----------------------------------------------------------------------------------------------
def vitvq_forward(sd: Dict[str, Tensor], img: Tensor, cfg: dict) -> Tuple[Tensor, Tensor, Tensor]:
    """ViTVQ.forward, vitvqgan.py:44-48,61-72: encoder -> pre_quant -> quantiser -> post_quant
    -> decoder.  ``sd`` uses the LightningModule's key names (encoder./decoder./quantizer./
    pre_quant./post_quant.).  Returns (reconstruction, quantiser loss, indices)."""
    p = cfg["patch_size"]
    g = cfg["image_size"] // p
    e, d, q = cfg["encoder"], cfg["decoder"], cfg["quantizer"]
    h = vit_encoder(sd, img, patch=p, depth=e["depth"], heads=e["heads"], prefix="encoder.")
    z = h @ sd["pre_quant.weight"].t() + sd["pre_quant.bias"]
    zq, qloss, idx = vq_forward(z, sd["quantizer.embedding.weight"], q.get("beta", 0.25),
                                q.get("use_residual", False), q.get("num_quantizers"))
    t = zq @ sd["post_quant.weight"].t() + sd["post_quant.bias"]
    rec = vit_decoder(sd, t, patch=p, depth=d["depth"], heads=d["heads"], grid_hw=(g, g), prefix="decoder.")
    return rec, qloss, idx


def vitvq_loss(sd: Dict[str, Tensor], img: Tensor, cfg: dict) -> Tuple[Tensor, Tensor, Tensor]:
    """loss = mean((rec - img)^2) + qloss, the fwd+bwd unit of SURVEY.md section 8d."""
    rec, qloss, idx = vitvq_forward(sd, img, cfg)
    return ((rec - img) ** 2).mean() + qloss, rec, idx


# ----------------------------------------------------------------------------------------------
# parameter construction (reference layers.py:71-82, quantizers.py:32-33, vitvqgan.py:35-39)
# ----------------------------------------------------------------------------------------------
def _xavier(shape, fan_out, fan_in, gen) -> Tensor:
    a = math.sqrt(6.0 / (fan_in + fan_out))
    return (torch.rand(shape, generator=gen) * 2 - 1) * a


def init_transformer_sd(prefix: str, dim: int, depth: int, heads: int, mlp_dim: int, dim_head: int,
                        gen: torch.Generator) -> Dict[str, Tensor]:
    inner = heads * dim_head
    sd: Dict[str, Tensor] = {}
    for i in range(depth):
        a, f = f"{prefix}layers.{i}.0.", f"{prefix}layers.{i}.1."
        sd[a + "norm.weight"], sd[a + "norm.bias"] = torch.ones(dim), torch.zeros(dim)
        sd[a + "fn.to_qkv.weight"] = _xavier((3 * inner, dim), 3 * inner, dim, gen)
        sd[a + "fn.to_out.weight"] = _xavier((dim, inner), dim, inner, gen)
        sd[a + "fn.to_out.bias"] = torch.zeros(dim)
        sd[f + "norm.weight"], sd[f + "norm.bias"] = torch.ones(dim), torch.zeros(dim)
        sd[f + "fn.net.0.weight"] = _xavier((mlp_dim, dim), mlp_dim, dim, gen)
        sd[f + "fn.net.0.bias"] = torch.zeros(mlp_dim)
        sd[f + "fn.net.2.weight"] = _xavier((dim, mlp_dim), dim, mlp_dim, gen)
        sd[f + "fn.net.2.bias"] = torch.zeros(dim)
    sd[prefix + "norm.weight"], sd[prefix + "norm.bias"] = torch.ones(dim), torch.zeros(dim)
    return sd


def init_vitvq_sd(cfg: dict, seed: int = 0) -> Dict[str, Tensor]:
    """Random-init weights with the reference's *distributions* (xavier-uniform matrices, zero
    Linear biases, unit LayerNorm, N(0,1) codebook; layers.py:71-82, quantizers.py:33).  The
    RNG stream is this oracle's own: parity tests share one state_dict between the oracle and
    the CUDA modules instead of re-deriving the reference's construction order."""
    gen = torch.Generator().manual_seed(seed)
    p, C = cfg["patch_size"], 3
    g = cfg["image_size"] // p
    e, d, q = cfg["encoder"], cfg["decoder"], cfg["quantizer"]
    sd: Dict[str, Tensor] = {}
    pd = C * p * p
    sd["encoder.en_pos_embedding"] = torch.from_numpy(sincos_pos_embed(e["dim"], (g, g))).unsqueeze(0)
    sd["encoder.to_patch_embedding.0.weight"] = _xavier((e["dim"], pd), e["dim"], pd, gen).reshape(e["dim"], C, p, p)
    sd["encoder.to_patch_embedding.0.bias"] = (torch.rand(e["dim"], generator=gen) * 2 - 1) / math.sqrt(pd)
    sd.update(init_transformer_sd("encoder.transformer.", e["dim"], e["depth"], e["heads"], e["mlp_dim"],
                                  e.get("dim_head", 64), gen))
    sd["decoder.de_pos_embedding"] = torch.from_numpy(sincos_pos_embed(d["dim"], (g, g))).unsqueeze(0)
    sd.update(init_transformer_sd("decoder.transformer.", d["dim"], d["depth"], d["heads"], d["mlp_dim"],
                                  d.get("dim_head", 64), gen))
    sd["decoder.to_pixel.1.weight"] = _xavier((d["dim"], pd), d["dim"], pd, gen).reshape(d["dim"], C, p, p)
    sd["decoder.to_pixel.1.bias"] = (torch.rand(C, generator=gen) * 2 - 1) / math.sqrt(pd)
    sd["quantizer.embedding.weight"] = torch.randn(q["n_embed"], q["embed_dim"], generator=gen)
    kq = 1.0 / math.sqrt(e["dim"])
    sd["pre_quant.weight"] = (torch.rand(q["embed_dim"], e["dim"], generator=gen) * 2 - 1) * kq
    sd["pre_quant.bias"] = (torch.rand(q["embed_dim"], generator=gen) * 2 - 1) * kq
    kp = 1.0 / math.sqrt(q["embed_dim"])
    sd["post_quant.weight"] = (torch.rand(d["dim"], q["embed_dim"], generator=gen) * 2 - 1) * kp
    sd["post_quant.bias"] = (torch.rand(d["dim"], generator=gen) * 2 - 1) * kp
    return sd


# configs of the reference (configs/imagenet_vitvq_{small,base,large}.yaml:7-19)
CONFIGS = {
    "small": dict(image_size=256, patch_size=8,
                  encoder=dict(dim=512, depth=8, heads=8, mlp_dim=2048),
                  decoder=dict(dim=512, depth=8, heads=8, mlp_dim=2048),
                  quantizer=dict(embed_dim=32, n_embed=8192)),
    "base": dict(image_size=256, patch_size=8,
                 encoder=dict(dim=768, depth=12, heads=12, mlp_dim=3072),
                 decoder=dict(dim=768, depth=12, heads=12, mlp_dim=3072),
                 quantizer=dict(embed_dim=32, n_embed=8192)),
    "base_rq4": dict(image_size=256, patch_size=8,
                     encoder=dict(dim=768, depth=12, heads=12, mlp_dim=3072),
                     decoder=dict(dim=768, depth=12, heads=12, mlp_dim=3072),
                     quantizer=dict(embed_dim=32, n_embed=8192, use_residual=True, num_quantizers=4)),
    "large": dict(image_size=256, patch_size=8,
                  encoder=dict(dim=512, depth=8, heads=8, mlp_dim=2048),
                  decoder=dict(dim=1280, depth=32, heads=16, mlp_dim=5120),
                  quantizer=dict(embed_dim=32, n_embed=8192)),
    # not a reference config: a miniature with the same structure for fast parity tests
    "tiny": dict(image_size=64, patch_size=8,
                 encoder=dict(dim=128, depth=2, heads=2, mlp_dim=256),
                 decoder=dict(dim=192, depth=2, heads=3, mlp_dim=384),
                 quantizer=dict(embed_dim=32, n_embed=512)),
}


def flops_per_image(cfg: dict) -> float:
    """Algorithmic forward FLOPs per image, BASELINE.md section 3 / SURVEY.md section 8d."""
    n = (cfg["image_size"] // cfg["patch_size"]) ** 2
    pd = 3 * cfg["patch_size"] ** 2
    q = cfg["quantizer"]

    def blk(c):
        D, inner, m = c["dim"], 64 * c["heads"], c["mlp_dim"]
        return 6 * D * inner + 4 * n * inner + 2 * inner * D + 4 * D * m
    e, d = cfg["encoder"], cfg["decoder"]
    T = q.get("num_quantizers") or 1 if q.get("use_residual") else 1
    per_tok = (e["depth"] * blk(e) + d["depth"] * blk(d) + 2 * pd * e["dim"] + 2 * pd * d["dim"]
               + 2 * e["dim"] * q["embed_dim"] + 2 * q["embed_dim"] * d["dim"]
               + T * 2 * q["embed_dim"] * q["n_embed"])
    return float(n * per_tok)


# the config of tests/golden/ref_vitvq_small.npz: residual VQ, unequal encoder / decoder depths, dim_head != dim / heads
SMALL_REF_CFG = dict(image_size=48, patch_size=8, encoder=dict(dim=64, depth=2, heads=2, mlp_dim=96, dim_head=32),
                     decoder=dict(dim=64, depth=1, heads=2, mlp_dim=64, dim_head=32),
                     quantizer=dict(embed_dim=32, n_embed=128, use_residual=True, num_quantizers=2))


def seeded_gumbel_softmax(seed: int):
    """a drop-in for F.gumbel_softmax (same formula as torch's) whose noise comes from a CPU generator seeded with `seed`:
    a run on any device draws the same noise, so a GPU module can be compared with a golden recorded on the CPU"""
    gen = torch.Generator().manual_seed(seed)

    def gumbel_softmax(logits, tau=1.0, hard=False, eps=1e-10, dim=-1):
        g = -torch.empty(logits.shape, dtype=torch.float32).exponential_(generator=gen).log()
        y = ((logits + g.to(device=logits.device, dtype=logits.dtype)) / tau).softmax(dim)
        if hard:
            index = y.max(dim, keepdim=True)[1]
            return torch.zeros_like(logits).scatter_(dim, index, 1.0) - y.detach() + y
        return y
    return gumbel_softmax


class _Golden(dict):
    @property
    def files(self):
        return list(self)


def load_golden(path: str) -> "_Golden":
    """np.load of `path` (an .npz) merged with its continuation files <stem>.1.npz, <stem>.2.npz, ...: a fixture larger
    than 1 MB is stored in several files.  Offers NpzFile's `.files` / `[key]` interface."""
    import os
    out = _Golden(np.load(path))
    stem = path[:-len(".npz")]
    i = 1
    while os.path.exists(f"{stem}.{i}.npz"):
        out.update(np.load(f"{stem}.{i}.npz"))
        i += 1
    return out


def save_golden(path: str, arrays: Dict[str, np.ndarray], limit: int = 900_000) -> None:
    """np.savez_compressed of `arrays` into `path` and as many continuation files as keep each under `limit` bytes of
    array data (the inverse of load_golden)"""
    parts, cur, size = [], {}, 0
    for k, v in arrays.items():
        if cur and size + v.nbytes > limit:
            parts.append(cur)
            cur, size = {}, 0
        cur[k] = v
        size += v.nbytes
    parts.append(cur)
    stem = path[:-len(".npz")]
    for i, part in enumerate(parts):
        np.savez_compressed(path if i == 0 else f"{stem}.{i}.npz", **part)
