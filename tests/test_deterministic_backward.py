"""CPU checks of the opt-in bit-reproducible backward: which `ops` function VectorQuantizeFn and stage2.TokenEmbedFn call
under the default, under torch.use_deterministic_algorithms(True) and under B200VQ_DETERMINISTIC (the `functional`
attribute it is read into), and the argument checks of the two deterministic C entry points, which run before any CUDA
call and so need no GPU."""
import os
import subprocess
import sys

import pytest
import torch

import enhancing_transformers_b200 as etb
from enhancing_transformers_b200 import functional as Fn
from enhancing_transformers_b200 import ops
from enhancing_transformers_b200 import stage2 as S2

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def spies(monkeypatch):
    """CPU stand-ins for the forward wrappers, and spies recording which backward wrapper ran"""
    calls = []

    def vq_fwd(z, E, depth, beta, use_norm=True):
        return z.clone(), z.sum() * 0, torch.zeros(z.shape[0], depth, dtype=torch.int64)

    def vq_spy(name):
        def bwd(z, E, idx, g_out, g_loss, residual, beta, use_norm=True):
            calls.append(name)
            return torch.zeros_like(z), torch.zeros_like(E)
        return bwd

    def token_embed_fwd(conds, codes, Wc, pos_c, Wi, pos_i):
        return torch.zeros(conds.shape[0] * (conds.shape[1] + codes.shape[1]), Wi.shape[1])

    def te_spy(name):
        def bwd(conds, codes, g, Vc, Vi):
            calls.append(name)
            C = g.shape[-1]
            return torch.zeros(Vc, C), torch.zeros(conds.shape[1], C), torch.zeros(Vi, C), torch.zeros(codes.shape[1], C)
        return bwd

    monkeypatch.setattr(ops, "vq_fwd", vq_fwd)
    monkeypatch.setattr(ops, "vq_bwd", vq_spy("vq_bwd"))
    monkeypatch.setattr(ops, "vq_bwd_deterministic", vq_spy("vq_bwd_deterministic"))
    monkeypatch.setattr(ops, "token_embed_fwd", token_embed_fwd)
    monkeypatch.setattr(ops, "token_embed_bwd", te_spy("token_embed_bwd"))
    monkeypatch.setattr(ops, "token_embed_bwd_deterministic", te_spy("token_embed_bwd_deterministic"))
    monkeypatch.setattr(Fn, "DETERMINISTIC", False)
    return calls


def _vq_step():
    z = torch.randn(8, 32, requires_grad=True)
    E = torch.randn(16, 32, requires_grad=True)
    out, loss, _ = Fn.VectorQuantizeFn.apply(z, E, 1, 0.25, False, True)
    return out.sum() + loss


def _token_embed_step():
    B, Tc, Ti, C = 2, 1, 4, 8
    Wc, Wi = torch.randn(3, C, requires_grad=True), torch.randn(5, C, requires_grad=True)
    pos_c, pos_i = torch.zeros(1, Tc, C, requires_grad=True), torch.zeros(1, Ti, C, requires_grad=True)
    conds, codes = torch.zeros(B, Tc, dtype=torch.int64), torch.zeros(B, Ti, dtype=torch.int64)
    return S2.TokenEmbedFn.apply(conds, codes, Wc, pos_c, Wi, pos_i).sum()


@pytest.mark.parametrize("step,name", [(_vq_step, "vq_bwd"), (_token_embed_step, "token_embed_bwd")])
def test_default_backward_keeps_the_atomic_path(spies, step, name):
    assert not torch.are_deterministic_algorithms_enabled()
    step().backward()
    assert spies == [name]


@pytest.mark.parametrize("step,name", [(_vq_step, "vq_bwd"), (_token_embed_step, "token_embed_bwd")])
def test_torch_deterministic_flag_selects_the_deterministic_path(spies, step, name):
    loss = step()                                    # forward outside the flag: the switch is read when backward runs
    torch.use_deterministic_algorithms(True)
    try:
        loss.backward()
    finally:
        torch.use_deterministic_algorithms(False)
    assert spies == [name + "_deterministic"]


@pytest.mark.parametrize("step,name", [(_vq_step, "vq_bwd"), (_token_embed_step, "token_embed_bwd")])
def test_env_switch_selects_the_deterministic_path(spies, monkeypatch, step, name):
    monkeypatch.setattr(Fn, "DETERMINISTIC", True)
    step().backward()
    monkeypatch.setattr(Fn, "DETERMINISTIC", False)
    step().backward()
    assert spies == [name + "_deterministic", name]


def test_env_variable_is_read_at_import():
    code = "import enhancing_transformers_b200.functional as F; print(F.DETERMINISTIC, F.deterministic())"
    for value, want in (("1", "True True"), ("0", "False False")):
        env = dict(os.environ, B200VQ_DETERMINISTIC=value)
        out = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=300)
        assert out.returncode == 0, out.stderr
        assert out.stdout.split() == want.split()


def test_deterministic_entry_points_reject_bad_arguments_before_touching_the_device():
    lib = etb._lib.lib()

    def err():
        return lib.b200vq_last_error().decode()
    fake = 256                                       # never dereferenced: every call below fails its argument checks
    M, K, D = 128, 256, 32
    ws = lib.b200vq_vq_bwd_deterministic_workspace_bytes(M, K, D, 4)
    assert ws >= M * 4 * D * 4                       # at least the per-entry contributions
    assert lib.b200vq_vq_bwd_deterministic_workspace_bytes(M, K, D, 9) == 0
    args = [fake] * 7 + [M, K, D, 4, 1, 0.25, 1, fake, ws, None]
    bad = list(args); bad[0] = None                  # z
    assert lib.b200vq_vq_bwd_deterministic(*bad) < 0 and "null pointer" in err()
    bad = list(args); bad[14] = None                 # workspace
    assert lib.b200vq_vq_bwd_deterministic(*bad) < 0 and "null pointer" in err()
    bad = list(args); bad[15] = ws - 1
    assert lib.b200vq_vq_bwd_deterministic(*bad) < 0 and "workspace too small" in err()
    bad = list(args); bad[10] = 9                    # depth
    assert lib.b200vq_vq_bwd_deterministic(*bad) < 0 and "num_quantizers" in err()
    bad = list(args); bad[10] = 0
    assert lib.b200vq_vq_bwd_deterministic(*bad) < 0 and "num_quantizers" in err()
    bad = list(args); bad[9] = 16                    # embed_dim
    assert lib.b200vq_vq_bwd_deterministic(*bad) < 0 and "embed_dim" in err()
    bad = list(args); bad[7] = 126                   # M % 4
    assert lib.b200vq_vq_bwd_deterministic(*bad) < 0 and "M % 4" in err()

    B, Tc, Ti, C, Vc, Vi = 4, 1, 64, 64, 10, 256
    ws = lib.b200vq_token_embed_bwd_deterministic_workspace_bytes(B, Tc, Ti, C, Vc, Vi)
    assert ws > 0
    args = [fake] * 7 + [B, Tc, Ti, C, Vc, Vi, fake, ws, None]
    bad = list(args); bad[1] = None                  # codes
    assert lib.b200vq_token_embed_bwd_deterministic(*bad) < 0 and "null pointer" in err()
    bad = list(args); bad[14] = ws - 1
    assert lib.b200vq_token_embed_bwd_deterministic(*bad) < 0 and "workspace too small" in err()
    bad = list(args); bad[12] = 0                    # Vi
    assert lib.b200vq_token_embed_bwd_deterministic(*bad) < 0 and "vocabulary" in err()
    bad = list(args); bad[7] = 0                     # B
    assert lib.b200vq_token_embed_bwd_deterministic(*bad) < 0 and "bad shape" in err()
