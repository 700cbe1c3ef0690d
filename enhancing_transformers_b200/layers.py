"""Drop-in ViTEncoder / ViTDecoder for the reference's ``enhancing/modules/stage1/layers.py``.

Same constructor keywords (``vitvqgan.py:35-36`` splats the YAML dicts into them), same
``forward`` signatures, same ``state_dict`` keys and shapes (checkpoints load both ways), same
sub-module tree (``transformer.layers[i][0].fn.to_qkv`` ...), but every FLOP runs in
libb200vq.so: the sub-modules are parameter containers whose ``forward`` dispatch to the CUDA
kernels, and ``Transformer.forward`` runs each pre-norm block as one fused autograd unit.

There is no CPU path: CPU tensors raise (use the reference classes on CPU)."""
from __future__ import annotations

import math
from typing import Tuple, Union

import numpy as np
import torch
import torch.nn as nn

from . import functional as Fn

Size2 = Union[Tuple[int, int], int]


def _pair(v: Size2) -> Tuple[int, int]:
    return v if isinstance(v, tuple) else (v, v)


def sincos_table(dim: int, grid_hw: Tuple[int, int]) -> np.ndarray:
    """Fixed 2-D sin-cos positional table, float64 math then cast to float32, as the reference
    builds it (layers.py:21-68): channels [0, dim/2) encode the column index, [dim/2, dim) the
    row index, each half laid out as [sin | cos] over frequencies 10000^(-j/(dim/4))."""
    assert dim % 4 == 0, "embedding dim must be divisible by 4 for the 2-D sin-cos table"
    gh, gw = grid_hw
    freq = 1.0 / (10000.0 ** (np.arange(dim // 4, dtype=np.float64) / (dim / 4.0)))
    cols = np.tile(np.arange(gw, dtype=np.float64), gh)          # column index of token (r, c)
    rows = np.repeat(np.arange(gh, dtype=np.float64), gw)
    parts = []
    for coord in (cols, rows):
        ang = coord[:, None] * freq[None, :]
        parts += [np.sin(ang), np.cos(ang)]
    return np.concatenate(parts, axis=1).astype(np.float32)


def _xavier_(w: torch.Tensor) -> None:
    flat = w.view(w.shape[0], -1)
    bound = math.sqrt(6.0 / (flat.shape[0] + flat.shape[1]))
    with torch.no_grad():
        w.uniform_(-bound, bound)


def _init_like_reference(module: nn.Module) -> None:
    """Same distributions as reference init_weights (layers.py:71-82): xavier-uniform matrices,
    zero Linear biases, unit LayerNorm; conv biases keep torch's default."""
    for m in module.modules():
        if isinstance(m, nn.Linear):
            _xavier_(m.weight)
            if m.bias is not None:
                nn.init.zeros_(m.bias)
        elif isinstance(m, nn.LayerNorm):
            nn.init.ones_(m.weight)
            nn.init.zeros_(m.bias)
        elif isinstance(m, (nn.Conv2d, nn.ConvTranspose2d)):
            _xavier_(m.weight)


def _flat2d(x: torch.Tensor) -> torch.Tensor:
    x = x.contiguous()
    return x.view(-1, x.shape[-1])


class PreNorm(nn.Module):
    """LayerNorm in front of a sub-block; parameter container (`norm`, `fn`) + stand-alone forward."""

    def __init__(self, dim: int, fn: nn.Module) -> None:
        super().__init__()
        self.norm, self.fn = nn.LayerNorm(dim), fn

    def forward(self, x: torch.Tensor, **kwargs) -> torch.Tensor:
        flat = _flat2d(x)
        normed = Fn.LayerNormFn.apply(flat, self.norm.weight, self.norm.bias, False)
        return self.fn(normed.view_as(x), **kwargs)


class FeedForward(nn.Module):
    """Linear -> Tanh -> Linear; `net.0` / `net.2` hold the weights (checkpoint keys)."""

    def __init__(self, dim: int, hidden_dim: int) -> None:
        super().__init__()
        up, down = nn.Linear(dim, hidden_dim), nn.Linear(hidden_dim, dim)
        self.net = nn.Sequential(up, nn.Tanh(), down)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        up, down = self.net[0], self.net[2]
        hidden = Fn.LinearFn.apply(_flat2d(x), up.weight, up.bias, 1, False)      # bias + tanh fused in the GEMM epilogue
        y = Fn.LinearFn.apply(hidden, down.weight, down.bias, 0, False)
        return y.view(*x.shape[:-1], -1)


class Attention(nn.Module):
    """Multi-head self-attention; `to_qkv` (no bias) and `to_out` hold the weights."""

    def __init__(self, dim: int, heads: int = 8, dim_head: int = 64) -> None:
        super().__init__()
        self.heads, self.dim_head = heads, dim_head
        self.scale = dim_head ** -0.5
        width = heads * dim_head
        self.attend = nn.Softmax(dim=-1)          # module-tree parity only; the kernel fuses the softmax
        self.to_qkv = nn.Linear(dim, 3 * width, bias=False)
        single_head_identity = heads == 1 and dim_head == dim
        self.to_out = nn.Identity() if single_head_identity else nn.Linear(width, dim)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        batch, tokens, _ = x.shape
        qkv = Fn.LinearFn.apply(_flat2d(x), self.to_qkv.weight, None, 0, False)
        ctx = Fn.AttentionCoreFn.apply(qkv, batch, tokens, self.heads, self.dim_head)
        if isinstance(self.to_out, nn.Linear):
            ctx = Fn.LinearFn.apply(ctx, self.to_out.weight, self.to_out.bias, 0, False)
        return ctx.view(batch, tokens, -1)


class Transformer(nn.Module):
    """`depth` pre-norm blocks + final LayerNorm; forward runs each block as one fused autograd unit."""

    def __init__(self, dim: int, depth: int, heads: int, dim_head: int, mlp_dim: int) -> None:
        super().__init__()
        blocks = [nn.ModuleList([PreNorm(dim, Attention(dim, heads=heads, dim_head=dim_head)),
                                 PreNorm(dim, FeedForward(dim, mlp_dim))]) for _ in range(depth)]
        self.layers = nn.ModuleList(blocks)
        self.norm = nn.LayerNorm(dim)
        self.heads, self.dim_head = heads, dim_head
        self.round_final = False    # decoder sets it: its final LN only feeds the to_pixel GEMM

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        batch, tokens, width = x.shape
        att0 = self.layers[0][0].fn if len(self.layers) else None
        if att0 is not None and not isinstance(att0.to_out, nn.Linear):
            # heads == 1 and dim_head == dim (reference layers.py:112,120: no output projection): the fused
            # stack always has a to_out GEMM, so run the sub-modules one by one (same kernels, stand-alone units)
            for pre_attn, pre_ff in self.layers:
                x = Fn.AddFn.apply(pre_attn(x), x)
                x = Fn.AddFn.apply(pre_ff(x), x)
            h = Fn.LayerNormFn.apply(_flat2d(x), self.norm.weight, self.norm.bias, self.round_final)
            return h.view(batch, tokens, width)
        params = []
        for pre_attn, pre_ff in self.layers:
            att, ff = pre_attn.fn, pre_ff.fn
            params += [pre_attn.norm.weight, pre_attn.norm.bias, att.to_qkv.weight, att.to_out.weight, att.to_out.bias,
                       pre_ff.norm.weight, pre_ff.norm.bias, ff.net[0].weight, ff.net[0].bias, ff.net[2].weight, ff.net[2].bias]
        h = Fn.TransformerFn.apply(_flat2d(x), batch, tokens, self.heads, self.dim_head, self.round_final,
                                   self.norm.weight, self.norm.bias, *params)
        return h.view(batch, tokens, width)


class QuantLinear(nn.Linear):
    """``pre_quant`` / ``post_quant`` of the unchanged ``ViTVQ`` (reference vitvqgan.py:38-39,63,69) on the
    tensor-core GEMM (gemm_tc.cu) instead of cuBLAS.  Same parameters and state-dict keys as the ``nn.Linear`` it replaces
    (`from_linear` shares them).  Always the error-compensated 3xTF32 product: ``pre_quant`` writes the
    vector whose nearest code is looked up, so its rounding decides the indices, and both GEMMs are
    memory-bound (K or N = 32) -- the extra tensor passes are free."""

    @classmethod
    def from_linear(cls, lin: nn.Linear) -> "QuantLinear":
        new = cls.__new__(cls)
        nn.Module.__init__(new)
        new.in_features, new.out_features = lin.in_features, lin.out_features
        new.weight, new.bias = lin.weight, lin.bias
        return new

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        y = Fn.LinearFn.apply(_flat2d(x), self.weight, self.bias, 0, True)
        return y.view(*x.shape[:-1], self.out_features)


class PosQuantLinear(QuantLinear):
    """``post_quant`` that also adds the decoder's positional table (SURVEY.md section 8f-1, opt-in through
    `etb.fuse_post_quant_pos`): one GEMM writes ``post_quant(z) + de_pos_embedding`` and the decoder skips its own add.
    The table stays the decoder's parameter (same state-dict key); this module only borrows a reference to it."""

    @classmethod
    def from_linear(cls, lin: nn.Linear, decoder: "ViTDecoder") -> "PosQuantLinear":
        new = super().from_linear(lin)
        object.__setattr__(new, "_decoder", decoder)          # not a child module: the decoder is registered once, by ViTVQ
        return new

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        table = self._decoder.de_pos_embedding
        tokens = table.shape[1]
        assert x.shape[-2] == tokens, "post_quant input must carry one row per decoder position"
        y = Fn.LinearPosFn.apply(_flat2d(x), self.weight, self.bias, table)
        return y.view(*x.shape[:-1], self.out_features)


class _Geometry:
    """image / patch bookkeeping shared by encoder and decoder (reference layers.py:157-166,189-198)"""

    def __init__(self, image_size: Size2, patch_size: Size2, channels: int) -> None:
        ih, iw = _pair(image_size)
        ph, pw = _pair(patch_size)
        assert ih % ph == 0 and iw % pw == 0, 'Image dimensions must be divisible by the patch size.'
        if pw % 4 or (channels * ph * pw) % 4:
            # the layout kernels move 16-byte pieces of a patch row and TMA needs 16-byte row strides of the im2col
            # matrix: a patch width that is not a multiple of 4 has no CUDA path here (every shipped config uses 8)
            raise NotImplementedError(f"b200vq: patch width must be a multiple of 4 (got {ph} x {pw}); "
                                      "use the reference modules for this geometry")
        self.image_hw = (ih, iw)
        self.patch = (ph, pw)
        self.grid = (ih // ph, iw // pw)
        self.num_patches = self.grid[0] * self.grid[1]
        self.patch_dim = channels * ph * pw

    def pos_table(self, dim: int) -> nn.Parameter:
        table = torch.from_numpy(sincos_table(dim, self.grid)).unsqueeze(0)
        return nn.Parameter(table, requires_grad=False)      # frozen, but part of the state dict like the reference's


class ViTEncoder(nn.Module):
    """reference layers.py:153-182: patch-embed conv (k = s = patch) + positional table + transformer"""

    def __init__(self, image_size: Size2, patch_size: Size2, dim: int, depth: int, heads: int, mlp_dim: int,
                 channels: int = 3, dim_head: int = 64) -> None:
        super().__init__()
        geo = _Geometry(image_size, patch_size, channels)
        self.num_patches, self.patch_dim, self.patch = geo.num_patches, geo.patch_dim, geo.patch
        conv = nn.Conv2d(channels, dim, kernel_size=patch_size, stride=patch_size)
        self.to_patch_embedding = nn.Sequential(conv, nn.Identity())     # index 0 keeps the checkpoint key
        self.en_pos_embedding = geo.pos_table(dim)
        self.transformer = Transformer(dim, depth, heads, dim_head, mlp_dim)
        _init_like_reference(self)

    def forward(self, img: torch.Tensor) -> torch.Tensor:
        conv = self.to_patch_embedding[0]
        tokens = Fn.PatchEmbedFn.apply(img.contiguous(), conv.weight, conv.bias, self.en_pos_embedding, self.patch)
        return self.transformer(tokens.view(img.shape[0], self.num_patches, -1))


class ViTDecoder(nn.Module):
    """reference layers.py:185-217: positional table + transformer + conv-transpose (k = s = patch) to pixels"""

    def __init__(self, image_size: Size2, patch_size: Size2, dim: int, depth: int, heads: int, mlp_dim: int,
                 channels: int = 3, dim_head: int = 64) -> None:
        super().__init__()
        geo = _Geometry(image_size, patch_size, channels)
        self.num_patches, self.patch_dim, self.patch, self.image_hw = geo.num_patches, geo.patch_dim, geo.patch, geo.image_hw
        self.transformer = Transformer(dim, depth, heads, dim_head, mlp_dim)
        self.transformer.round_final = True
        self.de_pos_embedding = geo.pos_table(dim)
        self.pos_added_upstream = False     # set by etb.fuse_post_quant_pos: post_quant's epilogue has already added the table
        deconv = nn.ConvTranspose2d(dim, channels, kernel_size=patch_size, stride=patch_size)
        self.to_pixel = nn.Sequential(nn.Identity(), deconv)             # index 1 keeps the checkpoint key
        _init_like_reference(self)

    def forward(self, token: torch.Tensor) -> torch.Tensor:
        batch, tokens, width = token.shape
        x = _flat2d(token) if self.pos_added_upstream else Fn.AddPosFn.apply(_flat2d(token), self.de_pos_embedding)
        x = self.transformer(x.view(batch, tokens, width))
        deconv = self.to_pixel[1]
        height, width_px = self.image_hw
        return Fn.ToPixelFn.apply(_flat2d(x), deconv.weight, deconv.bias, batch, height, width_px, self.patch)

    def get_last_layer(self) -> nn.Parameter:
        return self.to_pixel[-1].weight
