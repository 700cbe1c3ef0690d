"""Wide codebooks (embed_dim a multiple of 32 from 64 to 256), CPU side: the oracle against the reference's outputs
(tests/golden/vq_wide.npz, written by oracle/gen_golden_vq_wide.py), the D-aware workspace query and the C argument
checks for unsupported widths."""
import os

import numpy as np
import pytest
import torch

import enhancing_transformers_b200 as etb
from oracle import vitvq_oracle as O
from oracle.gen_golden_vq_wide import CASES

TAGS = [(tag, kw) for tag, _, kw in CASES] + [("d256.clustered", {})]


def _t(a):
    return torch.from_numpy(np.asarray(a))


@pytest.mark.parametrize("tag,kw", TAGS, ids=[t for t, _ in TAGS])
def test_quantizer_matches_reference(golden_dir, tag, kw, monkeypatch):
    g = O.load_golden(os.path.join(golden_dir, "vq_wide.npz"))
    kw = dict(kw)
    use_norm = kw.pop("use_norm", True)
    if not use_norm:                      # BaseQuantizer.norm is the identity (quantizers.py:24)
        monkeypatch.setattr(O, "l2norm", lambda x: x)
    z = _t(g[f"{tag}.z"]).requires_grad_(True)
    E = _t(g[f"{tag}.E"]).requires_grad_(True)
    out, loss, idx = O.vq_forward(z, E, 0.25, **kw)
    np.testing.assert_array_equal(idx.numpy(), g[f"{tag}.idx"])
    np.testing.assert_array_equal(out.detach().numpy(), g[f"{tag}.zq"])
    torch.testing.assert_close(loss.detach(), _t(g[f"{tag}.loss"]), rtol=1e-6, atol=0)
    g_out, g_loss = _t(g[f"{tag}.g_out"]), float(g[f"{tag}.g_loss"])
    ((out * g_out).sum() + loss * g_loss).backward()
    torch.testing.assert_close(z.grad, _t(g[f"{tag}.gz"]), rtol=1e-5, atol=1e-8)
    torch.testing.assert_close(E.grad, _t(g[f"{tag}.gE"]), rtol=1e-4, atol=1e-7)
    if use_norm:                          # the closed forms the kernels implement
        gz, gE = O.vq_backward_np(g[f"{tag}.z"], g[f"{tag}.E"], g[f"{tag}.idx"], g_out.numpy(), g_loss, 0.25,
                                  use_residual=bool(kw.get("use_residual")))
        np.testing.assert_allclose(gz, g[f"{tag}.gz"], rtol=2e-4, atol=1e-7)
        np.testing.assert_allclose(gE, g[f"{tag}.gE"], rtol=2e-3, atol=2e-7)
    if not kw and use_norm:
        D = g[f"{tag}.E"].shape[1]
        np.testing.assert_array_equal(O.vq_lookup_np(g[f"{tag}.z"].reshape(-1, D), g[f"{tag}.E"]).reshape(idx.shape),
                                      g[f"{tag}.idx"])


def test_forward_workspace_query():
    lib = etb._lib.lib()
    for M, K, depth in ((128, 256, 1), (4096, 8192, 4), (131072, 16384, 8), (132, 8, 2)):
        assert lib.b200vq_vq_fwd_workspace_bytes(M, K, 32, depth) == lib.b200vq_vq_workspace_bytes(M, K, depth)
    for D in (16, 48, 288):
        assert lib.b200vq_vq_fwd_workspace_bytes(4096, 8192, D, 1) == 0
        assert lib.b200vq_vq_fwd_ema_workspace_bytes(4096, 8192, D, 1, 0) == 0
        assert lib.b200vq_vq_bwd_deterministic_workspace_bytes(4096, 8192, D, 1) == 0
    # wide widths: the codebook transpose grows with D, the residual workspace appears with depth > 1
    w1 = lib.b200vq_vq_fwd_workspace_bytes(4096, 8192, 256, 1)
    assert w1 >= (256 * 8192 + 8192) * 4
    assert lib.b200vq_vq_fwd_workspace_bytes(4096, 8192, 256, 4) >= w1 + 4096 * 256 * 4
    assert lib.b200vq_vq_fwd_ema_workspace_bytes(4096, 8192, 256, 4, 1) > lib.b200vq_vq_fwd_ema_workspace_bytes(4096, 8192, 256, 4, 0)


@pytest.mark.parametrize("D", [48, 288])
def test_entry_points_reject_unsupported_widths_before_touching_the_device(D):
    lib = etb._lib.lib()

    def err():
        return lib.b200vq_last_error().decode()
    p, M, K = 256, 128, 256                                            # never dereferenced: validation comes first
    ws = 1 << 30
    assert lib.b200vq_vq_fwd(p, p, p, p, p, M, K, D, 1, 0.25, 1, p, ws, None) < 0 and "embed_dim" in err()
    assert lib.b200vq_vq_bwd(p, p, p, p, p, p, p, M, K, D, 1, 0, 0.25, 1, None) < 0 and "embed_dim" in err()
    assert lib.b200vq_vq_bwd_deterministic(p, p, p, p, p, p, p, M, K, D, 1, 0, 0.25, 1, p, ws, None) < 0 and "embed_dim" in err()
    assert lib.b200vq_vq_embed(p, p, p, M, K, D, 1, 1, None) < 0 and "embed_dim" in err()
    assert lib.b200vq_vq_fwd_ema(p, p, p, p, p, p, p, M, K, D, 1, 0.25, 1, 0, p, ws, None) < 0 and "embed_dim" in err()
    assert lib.b200vq_vq_ema_update(p, p, p, p, p, K, D, 0.99, 1e-5, None) < 0 and "embed_dim" in err()
