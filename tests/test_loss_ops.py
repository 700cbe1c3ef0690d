"""The loss stage's two native ops (SURVEY.md section 8f-2) against tests/golden/lossops.npz, which oracle/gen_golden.py
wrote from the REFERENCE's own CPU formulas (losses/op/upfirdn2d.py:168-206, losses/op/fused_act.py:110-122).
CPU tests pin the module's CPU branch; `-m gpu` tests run the sm_90a kernels through the C ABI (values, first-order
gradients and the double-backward an R1-style penalty needs)."""
import os

import numpy as np
import pytest
import torch

from enhancing_transformers_b200 import loss_ops as L


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, "lossops.npz"))


def _t(a, dev):
    return torch.from_numpy(np.asarray(a)).to(dev)


def _check_upfirdn2d(gold, dev):
    x, k = _t(gold["up.x"], dev), _t(gold["up.kernel"], dev)
    i = 0
    while f"up.{i}.cfg" in gold.files:
        u, d, *pad = (int(v) for v in gold[f"up.{i}.cfg"])
        xi = x.clone().requires_grad_(True)
        y = L.upfirdn2d(xi, k, up=u, down=d, pad=tuple(pad))
        np.testing.assert_allclose(y.detach().cpu().numpy(), gold[f"up.{i}.y"], rtol=1e-5, atol=1e-6)
        gx, = torch.autograd.grad((y * _t(gold[f"up.{i}.w"], dev)).sum(), xi)
        np.testing.assert_allclose(gx.cpu().numpy(), gold[f"up.{i}.gx"], rtol=1e-5, atol=1e-6)
        i += 1
    assert i == 8
    xi = x.clone().requires_grad_(True)
    y = L.upfirdn2d(xi, _t(gold["up.asym.kernel"], dev), up=2, down=1, pad=(1, 2, 2, 1))
    np.testing.assert_allclose(y.detach().cpu().numpy(), gold["up.asym.y"], rtol=1e-5, atol=1e-6)
    gx, = torch.autograd.grad((y * _t(gold["up.asym.w"], dev)).sum(), xi)
    np.testing.assert_allclose(gx.cpu().numpy(), gold["up.asym.gx"], rtol=1e-5, atol=1e-6)


def _check_bias_act(gold, dev):
    for tag in ("4d", "2d"):
        for use_b in (True, False):
            key = f"act.{tag}.{'b' if use_b else 'nob'}"
            x = _t(gold[f"act.{tag}.x"], dev).requires_grad_(True)
            b = _t(gold[f"act.{tag}.bias"], dev).requires_grad_(True)
            y = L.fused_leaky_relu(x, b if use_b else None)
            np.testing.assert_allclose(y.detach().cpu().numpy(), gold[key + ".y"], rtol=1e-6, atol=1e-7)
            grads = torch.autograd.grad((y * _t(gold[key + ".w"], dev)).sum(), [x] + ([b] if use_b else []), create_graph=True)
            np.testing.assert_allclose(grads[0].detach().cpu().numpy(), gold[key + ".gx"], rtol=1e-6, atol=1e-7)
            if use_b:
                np.testing.assert_allclose(grads[1].detach().cpu().numpy(), gold[key + ".gb"], rtol=1e-5, atol=1e-6)
            # double backward (gradient penalty): d/dw of <gx, v> = mask * scale * v, independent of x almost everywhere
            v = _t(gold[key + ".v"], dev)
            w = _t(gold[key + ".w"], dev).requires_grad_(True)
            y2 = L.fused_leaky_relu(x, b if use_b else None)
            gx2, = torch.autograd.grad((y2 * w).sum(), x, create_graph=True)
            gw, = torch.autograd.grad((gx2 * v).sum(), w)
            pre = x.detach() + (b.detach().view(1, -1, *([1] * (x.ndim - 2))) if use_b else 0)
            expect = torch.where(pre > 0, torch.ones_like(pre), torch.full_like(pre, 0.2)) * (2 ** 0.5) * v
            np.testing.assert_allclose(gw.cpu().numpy(), expect.cpu().numpy(), rtol=1e-6, atol=1e-7)


def test_upfirdn2d_cpu_branch_matches_reference_golden(gold):
    _check_upfirdn2d(gold, "cpu")


def test_fused_leaky_relu_cpu_branch_matches_reference_golden(gold):
    _check_bias_act(gold, "cpu")


def test_install_as_reference_ops_registers_the_package():
    import sys
    saved = {k: sys.modules.get(k) for k in ("enhancing.losses.op", "enhancing.losses.op.conv2d_gradfix")}
    try:
        mod = L.install_as_reference_ops()
        from importlib import import_module
        assert import_module("enhancing.losses.op") is mod
        for name in ("FusedLeakyReLU", "fused_leaky_relu", "upfirdn2d", "conv2d_gradfix"):     # losses/layers.py:19
            assert hasattr(mod, name)
        y = mod.FusedLeakyReLU(4)(torch.randn(2, 4, 3, 3))
        assert y.shape == (2, 4, 3, 3)
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


@pytest.mark.gpu
def test_upfirdn2d_kernel_matches_reference_golden(gold):
    _check_upfirdn2d(gold, "cuda")


@pytest.mark.gpu
def test_fused_leaky_relu_kernel_matches_reference_golden(gold):
    _check_bias_act(gold, "cuda")


@pytest.mark.gpu
def test_blur_layer_shape_at_discriminator_size():
    """the Blur of a 256 x 256 StyleDiscriminator stage (losses/layers.py:214-243): pad (2, 2) then stride-2 conv"""
    k1 = torch.tensor([1.0, 3.0, 3.0, 1.0])
    k = (k1[None] * k1[:, None] / 64).cuda()
    x = torch.randn(4, 64, 256, 256, device="cuda")
    y = L.upfirdn2d(x, k, pad=(2, 2))
    assert y.shape == (4, 64, 257, 257)
    ref = L.upfirdn2d_native(x[:1, :2].cpu(), k.cpu(), 1, 1, 1, 1, 2, 2, 2, 2)
    np.testing.assert_allclose(y[:1, :2].cpu().numpy(), ref.numpy(), rtol=1e-5, atol=1e-6)
