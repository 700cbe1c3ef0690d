"""Drop-in VectorQuantizer for the reference's ``enhancing/modules/stage1/quantizers.py``.

Same constructor (``VectorQuantizer(embed_dim, n_embed, beta=0.25, use_norm=True,
use_residual=False, num_quantizers=None, **kwargs)``, quantizers.py:67-68), same return triple
``(z_q with straight-through gradient, loss, int64 indices)`` and the attributes the unchanged
LightningModule reads (``embedding``, ``norm``, ``use_residual`` -- vitvqgan.py:82-85).  The
residual mode the task calls "ResidualQuantizer" is ``use_residual=True, num_quantizers=T``
exactly as in the reference (there is no separate class there, SURVEY.md fact #1).

Forward and backward each run as one fused CUDA launch sequence (csrc/vq.cu); the
[tokens, n_embed] distance matrix of quantizers.py:78-80 is never materialised.  ``embed_dim`` may be any
multiple of 32 from 32 to 256 (RQ-VAE quantises 256-wide features); other widths construct, as in the
reference, and are rejected by the first forward."""
from __future__ import annotations

import math
from functools import partial
from typing import Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import functional as Fn
from . import ops


class BaseQuantizer(nn.Module):
    def __init__(self, embed_dim: int, n_embed: int, straight_through: bool = True, use_norm: bool = True,
                 use_residual: bool = False, num_quantizers: Optional[int] = None) -> None:
        super().__init__()
        self.straight_through = straight_through
        self.use_norm = use_norm
        self.norm = (lambda x: F.normalize(x, dim=-1)) if use_norm else (lambda x: x)
        self.use_residual = use_residual
        self.num_quantizers = num_quantizers
        self.embed_dim = embed_dim
        self.n_embed = n_embed
        self.embedding = nn.Embedding(self.n_embed, self.embed_dim)
        self.embedding.weight.data.normal_()


class VectorQuantizer(BaseQuantizer):
    def __init__(self, embed_dim: int, n_embed: int, beta: float = 0.25, use_norm: bool = True,
                 use_residual: bool = False, num_quantizers: Optional[int] = None, **kwargs) -> None:
        super().__init__(embed_dim, n_embed, True, use_norm, use_residual, num_quantizers)
        self.beta = beta
        if use_residual and not num_quantizers:
            raise ValueError("use_residual=True needs num_quantizers")

    @property
    def depth(self) -> int:
        return int(self.num_quantizers) if self.use_residual else 1

    def forward(self, z: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        zc = z.contiguous()
        out, loss, idx = Fn.VectorQuantizeFn.apply(zc.view(-1, self.embed_dim), self.embedding.weight, self.depth,
                                                   float(self.beta), bool(self.use_residual), bool(self.use_norm))
        out = out.view_as(zc)
        idx = idx.view(*z.shape[:-1], self.depth) if self.use_residual else idx.view(*z.shape[:-1])
        return out, loss, idx

    def quantize(self, z: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """single-depth lookup (quantizers.py:74-92): (normalised code, loss, indices).  Inference helper:
        the returned code carries no autograd graph; training goes through forward()."""
        zc = z.detach().contiguous().view(-1, self.embed_dim)
        _, loss, idx = ops.vq_fwd(zc, self.embedding.weight.detach(), 1, float(self.beta), bool(self.use_norm))
        q = ops.vq_embed(self.embedding.weight.detach(), idx, 1, bool(self.use_norm)).view_as(z)
        return q, loss, idx.view(*z.shape[:-1])

    def embed_codes(self, code: torch.Tensor) -> torch.Tensor:
        """decode_codes fast path (vitvqgan.py:81-86 in one kernel): sum_t normalize(E[code[..., t]])"""
        depth = self.depth
        lead = code.shape[:-1] if self.use_residual else code.shape
        return ops.vq_embed(self.embedding.weight.detach(), code.contiguous().view(-1, depth), depth,
                            bool(self.use_norm)).view(*lead, self.embed_dim)


class EMAVectorQuantizer(VectorQuantizer):
    """VectorQuantizer whose codebook is trained by exponential moving averages instead of gradients (van den Oord et al.
    2017, appendix A.1, in the form of Taming Transformers' ``EMAVectorQuantizer``; RQ-VAE trains its shared codebook the
    same way).  Same constructor plus ``decay`` and ``eps``, same lookup, codes and straight-through value; the loss is
    ``beta * mean((sg(q) - norm(z))^2)`` (averaged over the depths in residual mode) without a codebook term, and
    ``embedding.weight`` is frozen (``requires_grad = False``).

    Every forward in training mode (``self.training``; grad mode does not matter) gathers, over all tokens and depths, the
    count ``n_k`` and the sum ``s_k`` of the vectors the lookup compared per code, sums them over ``process_group`` (default:
    WORLD) when torch.distributed runs with more than one rank -- one all-reduce of one flat fp32 buffer -- and then updates,
    on the device::

        cluster_size <- decay * cluster_size + (1 - decay) * n
        embed_avg    <- decay * embed_avg    + (1 - decay) * s
        weight_k      = embed_avg_k / ((cluster_size_k + eps) / (N + K * eps) * N),   N = sum_k cluster_size_k

    The backward uses the codebook the forward looked up in.  Eval mode: the same lookup and loss, no update.  The buffers
    ``cluster_size`` and ``embed_avg`` join VectorQuantizer's state-dict keys; a state dict without them (a gradient-trained
    checkpoint) re-seeds them from the loaded weight as the constructor does."""

    def __init__(self, embed_dim: int, n_embed: int, beta: float = 0.25, use_norm: bool = True,
                 use_residual: bool = False, num_quantizers: Optional[int] = None, decay: float = 0.99, eps: float = 1e-5,
                 **kwargs) -> None:
        super().__init__(embed_dim, n_embed, beta, use_norm, use_residual, num_quantizers, **kwargs)
        self.decay = decay
        self.eps = eps
        self.embedding.weight.requires_grad_(False)
        self.register_buffer("cluster_size", torch.zeros(n_embed))
        self.register_buffer("embed_avg", self.embedding.weight.detach().clone())
        self.process_group = None

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        super()._load_from_state_dict(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs)
        w = state_dict.get(prefix + "embedding.weight")
        if w is None or tuple(w.shape) != tuple(self.embed_avg.shape):
            return
        with torch.no_grad():          # otherwise the first update would overwrite the loaded codebook
            if prefix + "embed_avg" not in state_dict:
                self.embed_avg.copy_(w)
            if prefix + "cluster_size" not in state_dict:
                self.cluster_size.zero_()

    def forward(self, z: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        zc = z.contiguous()
        weight = self.embedding.weight
        update = self.training
        # the update rewrites the weight in place, which autograd's version counter does not see: the backward gets a copy
        E = weight.detach().clone() if update and torch.is_grad_enabled() else weight.detach()
        res = Fn.EMAVectorQuantizeFn.apply(zc.view(-1, self.embed_dim), E, self.depth, float(self.beta), bool(self.use_residual),
                                           bool(self.use_norm), update)
        out, loss, idx = res[:3]
        if update:
            self._update(res[3])
        out = out.view_as(zc)
        idx = idx.view(*z.shape[:-1], self.depth) if self.use_residual else idx.view(*z.shape[:-1])
        return out, loss, idx

    def _update(self, stats: torch.Tensor) -> None:
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_world_size(self.process_group) > 1:
            dist.all_reduce(stats, op=dist.ReduceOp.SUM, group=self.process_group)
        ops.vq_ema_update(stats, self.cluster_size, self.embed_avg, self.embedding.weight.data, self.decay, self.eps)


class GumbelQuantizer(BaseQuantizer):
    """Drop-in for the reference's ``GumbelQuantizer`` (quantizers.py:95-126; used by ``ViTVQGumbel``, vitvqgan.py:147-176).

    Same constructor and the same ``(z_q, kl-to-uniform loss, indices)`` triple.  The two contractions -- the
    [tokens, n_embed] logit matrix ``-|z|^2 - |e|^2 + 2 z e^T`` and ``soft_one_hot @ codebook`` -- run on the tensor-core GEMM
    (3xTF32: the logits feed a softmax with temperature, so they keep fp32-grade accuracy); the Gumbel noise, the softmax
    and the KL term are PyTorch (``F.gumbel_softmax`` draws from the same generator as the reference, so a seeded run
    reproduces the reference's samples up to the rounding of the logits).  Unlike the arg-min lookup this quantiser is
    stochastic -- in eval mode too (hard one-hot of a noisy arg-max) -- so parity with the reference is distributional,
    not bit-wise (tests/test_gpu_model.py::test_gumbel_quantizer_matches_reference)."""

    def __init__(self, embed_dim: int, n_embed: int, temp_init: float = 1.0, use_norm: bool = True,
                 use_residual: bool = False, num_quantizers: Optional[int] = None, **kwargs) -> None:
        super().__init__(embed_dim, n_embed, False, use_norm, use_residual, num_quantizers)
        self.temperature = temp_init

    def quantize(self, z: torch.Tensor, temp: Optional[float] = None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        hard = not self.training            # the reference forces a hard sample in eval mode (quantizers.py:105-106)
        temp = self.temperature if temp is None else temp
        zn = self.norm(z.reshape(-1, self.embed_dim)).contiguous()
        en = self.norm(self.embedding.weight).contiguous()
        dots = Fn.LinearFn.apply(zn, en, None, 0, True)                                   # [tokens, n_embed]
        logits = 2.0 * dots - zn.pow(2).sum(dim=1, keepdim=True) - en.pow(2).sum(dim=1)
        logits = logits.view(*z.shape[:-1], -1)
        soft_one_hot = F.gumbel_softmax(logits, tau=temp, dim=-1, hard=hard)
        z_q = Fn.LinearFn.apply(soft_one_hot.reshape(-1, self.n_embed).contiguous(), en.t().contiguous(), None, 0, True)
        z_q = z_q.view(*z.shape[:-1], self.embed_dim)
        logp = F.log_softmax(logits, dim=-1)
        loss = torch.sum(logp.exp() * (logp + math.log(self.n_embed)), dim=-1).mean()
        return z_q, loss, soft_one_hot.argmax(dim=-1)

    def forward(self, z: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """quantizers.py:38-63 with straight_through = False: z_q carries the gradient of the soft sample"""
        if not self.use_residual:
            return self.quantize(z)
        z_q = torch.zeros_like(z)
        residual = z.detach().clone()
        losses, codes = [], []
        for _ in range(int(self.num_quantizers)):
            z_qi, loss, idx = self.quantize(residual.clone())
            residual = residual - z_qi          # like the reference's in-place sub_: later stages back-propagate into earlier samples
            z_q = z_q + z_qi
            codes.append(idx)
            losses.append(loss)
        losses, codes = map(partial(torch.stack, dim=-1), (losses, codes))
        return z_q, losses.mean(), codes
