"""ctypes binding of libb200vq.so (include/b200vq.h).  There is no fallback: if the library is
missing or a call fails, a RuntimeError is raised -- the product path never computes on the CPU."""
import ctypes
import os
import subprocess
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B200VQ_LIB") or os.path.join(_HERE, "libb200vq.so")   # B200VQ_LIB: development builds (trace hooks)
_lock = threading.Lock()
_lib = None

c_f = ctypes.c_void_p          # device pointers travel as integers
c_i, c_ll, c_sz, c_fl = ctypes.c_int, ctypes.c_longlong, ctypes.c_size_t, ctypes.c_float

_SIGNATURES = {
    "b200vq_version": (c_i, []),
    "b200vq_last_error": (ctypes.c_char_p, []),
    "b200vq_arch": (ctypes.c_char_p, []),
    "b200vq_launch_count": (c_ll, []),
    "b200vq_set_sm_limit": (c_i, [c_i]),
    "b200vq_gemm_tf32": (c_i, [c_f, c_ll, c_i, c_f, c_ll, c_i, c_f, c_ll, c_i, c_i, c_i, c_i, c_ll, c_f, c_f, c_ll, c_i,
                               c_f, c_ll, c_f, c_i, c_i, c_i, c_i, c_f]),
    "b200vq_gemm_3xtf32": (c_i, [c_f, c_f, c_ll, c_i, c_f, c_f, c_ll, c_i, c_f, c_ll, c_i, c_i, c_i, c_i, c_ll, c_f, c_f, c_ll,
                                 c_i, c_f, c_ll, c_f, c_i, c_i, c_i, c_f]),
    "b200vq_gemm_f16": (c_i, [c_f, c_ll, c_i, c_f, c_ll, c_i, c_f, c_ll, c_i, c_i, c_i, c_i, c_i, c_ll, c_f, c_f, c_ll, c_i,
                              c_f, c_ll, c_f, c_i, c_i, c_f, c_i, c_i, c_f]),
    "b200vq_splitk_reduce": (c_i, [c_f, c_i, c_ll, c_ll, c_f, c_f, c_f]),
    "b200vq_layernorm_fwd": (c_i, [c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_i, c_i, c_i, c_f]),
    "b200vq_layernorm_bwd_workspace_bytes": (c_sz, [c_i]),
    "b200vq_layernorm_bwd": (c_i, [c_f, c_i, c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_i, c_i, c_i, c_f, c_sz, c_f]),
    "b200vq_attention_fwd": (c_i, [c_f, c_f, c_i, c_f, c_i, c_i, c_i, c_i, c_fl, c_i, c_f]),
    "b200vq_attention_bwd": (c_i, [c_f, c_f, c_i, c_f, c_f, c_f, c_i, c_f, c_f, c_i, c_i, c_i, c_i, c_fl, c_i, c_f]),
    "b200vq_attention_f16_fwd": (c_i, [c_f, c_f, c_f, c_i, c_i, c_i, c_i, c_fl, c_f]),
    "b200vq_attention_f16_bwd": (c_i, [c_f, c_f, c_f, c_f, c_f, c_f, c_i, c_i, c_i, c_i, c_fl, c_f]),
    "b200vq_attention_exact_fwd": (c_i, [c_f, c_f, c_f, c_i, c_i, c_i, c_i, c_fl, c_f]),
    "b200vq_attention_exact_bwd": (c_i, [c_f, c_f, c_f, c_f, c_f, c_f, c_i, c_i, c_i, c_i, c_fl, c_f]),
    "b200vq_vq_workspace_bytes": (c_sz, [c_i, c_i, c_i]),
    "b200vq_vq_fwd_workspace_bytes": (c_sz, [c_i, c_i, c_i, c_i]),
    "b200vq_vq_fwd": (c_i, [c_f, c_f, c_f, c_f, c_f, c_i, c_i, c_i, c_i, c_fl, c_i, c_f, c_sz, c_f]),
    "b200vq_vq_bwd": (c_i, [c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_i, c_i, c_i, c_i, c_i, c_fl, c_i, c_f]),
    "b200vq_vq_bwd_deterministic_workspace_bytes": (c_sz, [c_i, c_i, c_i, c_i]),
    "b200vq_vq_bwd_deterministic": (c_i, [c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_i, c_i, c_i, c_i, c_i, c_fl, c_i, c_f, c_sz, c_f]),
    "b200vq_vq_embed": (c_i, [c_f, c_f, c_f, c_i, c_i, c_i, c_i, c_i, c_f]),
    "b200vq_vq_fwd_ema_workspace_bytes": (c_sz, [c_i, c_i, c_i, c_i, c_i]),
    "b200vq_vq_fwd_ema": (c_i, [c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_i, c_i, c_i, c_i, c_fl, c_i, c_i, c_f, c_sz, c_f]),
    "b200vq_vq_ema_update": (c_i, [c_f, c_f, c_f, c_f, c_f, c_i, c_i, c_fl, c_fl, c_f]),
    "b200vq_patchify": (c_i, [c_f, c_f, c_i, c_i, c_i, c_i, c_i, c_i, c_i, c_f]),
    "b200vq_unpatchify": (c_i, [c_f, c_f, c_f, c_i, c_i, c_i, c_i, c_i, c_i, c_f]),
    "b200vq_colsum_workspace_bytes": (c_sz, [c_i]),
    "b200vq_colsum": (c_i, [c_f, c_ll, c_i, c_i, c_f, c_f, c_sz, c_f]),
    "b200vq_round_tf32": (c_i, [c_f, c_f, c_ll, c_f]),
    "b200vq_add_rows_mod": (c_i, [c_f, c_f, c_f, c_ll, c_i, c_i, c_f]),
    "b200vq_split_tf32_lo": (c_i, [c_f, c_f, c_ll, c_f]),
    "b200vq_to_half": (c_i, [c_f, c_f, c_ll, c_f, c_f]),
    "b200vq_grad_scale_workspace_bytes": (c_sz, []),
    "b200vq_grad_scale": (c_i, [c_f, c_ll, c_i, c_f, c_f, c_sz, c_f]),
    "b200vq_bias_act": (c_i, [c_f, c_f, c_f, c_f, c_ll, c_i, c_i, c_i, c_i, c_fl, c_fl, c_f]),
    "b200vq_upfirdn2d": (c_i, [c_f, c_f, c_f, c_ll, c_i, c_i, c_i, c_i, c_i, c_i, c_i, c_i, c_i, c_i, c_i, c_i, c_f]),
    "b200vq_attention_causal_fwd": (c_i, [c_f, c_f, c_f, c_i, c_i, c_i, c_i, c_fl, c_i, c_i, c_i, c_f]),
    "b200vq_attention_causal_bwd": (c_i, [c_f, c_f, c_f, c_f, c_f, c_f, c_i, c_i, c_i, c_i, c_fl, c_i, c_i, c_i, c_f]),
    "b200vq_time_mix_fwd": (c_i, [c_f, c_f, c_f, c_ll, c_i, c_i, c_i, c_f]),
    "b200vq_time_mix_bwd_workspace_bytes": (c_sz, [c_ll, c_i]),
    "b200vq_time_mix_bwd": (c_i, [c_f, c_f, c_f, c_f, c_f, c_ll, c_i, c_i, c_f]),
    "b200vq_sqrelu": (c_i, [c_f, c_f, c_f, c_ll, c_i, c_i, c_f]),
    "b200vq_token_embed_fwd": (c_i, [c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_i, c_i, c_i, c_i, c_i, c_i, c_f]),
    "b200vq_token_embed_bwd": (c_i, [c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_i, c_i, c_i, c_i, c_i, c_i, c_f]),
    "b200vq_token_embed_bwd_deterministic_workspace_bytes": (c_sz, [c_i, c_i, c_i, c_i, c_i, c_i]),
    "b200vq_token_embed_bwd_deterministic": (c_i, [c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_i, c_i, c_i, c_i, c_i, c_i, c_f, c_sz, c_f]),
    "b200vq_copy_rows": (c_i, [c_f, c_f, c_i, c_i, c_i, c_i, c_i, c_i, c_i, c_f]),
    "b200vq_decode_attention": (c_i, [c_f, c_f, c_f, c_f, c_i, c_i, c_i, c_i, c_i, c_fl, c_f]),
    "b200vq_short_attention_fwd": (c_i, [c_f, c_f, c_ll, c_i, c_i, c_i, c_i, c_fl, c_f]),
    "b200vq_short_attention_bwd": (c_i, [c_f, c_f, c_f, c_ll, c_i, c_i, c_i, c_i, c_fl, c_f]),
    "b200vq_rq_embed_fwd": (c_i, [c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_i, c_i, c_i, c_i, c_i, c_i, c_i, c_f]),
    "b200vq_rq_embed_bwd": (c_i, [c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_i, c_i, c_i, c_i, c_i, c_i, c_i, c_f]),
    "b200vq_rq_embed_bwd_deterministic_workspace_bytes": (c_sz, [c_i, c_i, c_i, c_i, c_i, c_i, c_i]),
    "b200vq_rq_embed_bwd_deterministic": (c_i, [c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_i, c_i, c_i, c_i, c_i, c_i, c_i, c_f, c_sz, c_f]),
    "b200vq_rq_depth_input_fwd": (c_i, [c_f, c_f, c_f, c_f, c_f, c_ll, c_i, c_i, c_i, c_f]),
    "b200vq_rq_depth_input_bwd": (c_i, [c_f, c_f, c_f, c_f, c_f, c_ll, c_i, c_i, c_i, c_f]),
    "b200vq_rq_depth_input_bwd_deterministic_workspace_bytes": (c_sz, [c_ll, c_i, c_i, c_i]),
    "b200vq_rq_depth_input_bwd_deterministic": (c_i, [c_f, c_f, c_f, c_f, c_f, c_ll, c_i, c_i, c_i, c_f, c_sz, c_f]),
    "b200vq_code_sum_embed": (c_i, [c_f, c_ll, c_i, c_f, c_f, c_f, c_i, c_i, c_i, c_f]),
}
EXPORTS = tuple(_SIGNATURES)


def build(verbose: bool = False) -> str:
    """Compile csrc/*.cu for sm_90a into libb200vq.so (in-tree, next to this file)."""
    cmd = ["make", "-C", os.path.join(_HERE, "csrc"), "-j8"]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("building libb200vq.so failed:\n" + res.stdout[-4000:] + res.stderr[-4000:])
    if verbose:
        print(res.stdout[-2000:])
    return LIB_PATH


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        with _lock:
            if _lib is None:
                if not os.path.exists(LIB_PATH):
                    raise RuntimeError(
                        f"{LIB_PATH} not found: the CUDA extension is required (no CPU fallback). "
                        "Build it with `python -c 'import __graft_entry__ as g; g.build()'` or "
                        "`make -C enhancing_transformers_b200/csrc`.")
                handle = ctypes.CDLL(LIB_PATH)
                for name, (res, args) in _SIGNATURES.items():
                    fn = getattr(handle, name)      # AttributeError here == header/.so mismatch
                    fn.restype, fn.argtypes = res, args
                _lib = handle
    return _lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        raise RuntimeError(f"libb200vq {what} failed ({rc}): {lib().b200vq_last_error().decode()}")
