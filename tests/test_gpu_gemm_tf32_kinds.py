"""The tf32 and 3xTF32 GEMM kinds (mma.sync m16n8k8), element by element.

The fp32 data paths run on these kinds: the 3xTF32 product carries the patch embedding, to_pixel, pre_quant and
post_quant of every precision mode, and the tf32 / parity modes and the stage-2 GPT run all their GEMMs on them.

Exact checks.  Every output element of these kinds sees the same fragment values in the same k order whatever the
operand layout (tile_off changes only the address a value is loaded from), the tile width (BN changes only which warp
owns a column) or the CTA that runs the tile (the persistent schedule changes only that).  So the four (a_major,
b_major) layouts, BN 64 and BN 128, the full grid and a grid capped at CAPPED_CTAS CTAs (each running 8 or more tiles
back to back), a contiguous operand and a view of a wider buffer, and slice z of a split-K product and that slice run
alone must all give the same bits.  None of these needs a tolerance.

fp64 checks.  Inputs are N(0, 1) with row i of A scaled by 2^r_i and row j of B by 2^s_j, r and s uniform in
[-8, 8]: a power of two does not change how a value rounds to tf32, so an error in a small row or column is as visible
as one in a large one.  With S_ij = (|A| |B|^T)_ij over the stored operands, every element must satisfy

    |C_ij - ref_ij| <= tau * S_ij * g_ij + eps_ij

where ref is the epilogue applied in fp64, in the header's order, to the exact product of the stored operands; g_ij is
the factor the epilogue multiplies the product's error by (1 - aux^2 for tanh', at most 1 for tanh, else 1); eps_ij
covers the fp32 roundings of the added terms (2^-24 of each partial result, taken as 2^-23 so that it also covers the
gap between the computed and the exact partial result) and fast_tanh's absolute error (ex2.approx 2^-22 relative,
rcp.approx 2^-23, two 2^-24 roundings: below 6e-7).  tau comes from how the kernels compute, not from measured errors:

  tf32, operands rounded to tf32 where they are produced: each product of two tf32 values is exact in fp32.  An
  m16n8k8 step adds 8 products to the running sum, aligning the 9 terms to the largest and truncating; that loses at
  most one ulp (2^-23 relative) of the largest term per term, and no term exceeds S_ij.  K / 8 steps lose at most
  (9/8) K 2^-23 S_ij, so tau = K 2^-22.

  3xTF32 (lo = x - trunc_tf32(x), |lo| < 2^-10 |x|; the tensor core reads B in the A_lo pass and A in the B_lo pass as
  their truncated hi parts): per product, the tensor core's truncation of A_lo and of B_lo costs 2^-20 |a||b| each and
  the dropped A_lo B_lo term 2^-20 |a||b|, 3 2^-20 in all.  Each k-block of each pass is summed from zero over 4 steps
  (the bound above on 32 products: 2^-17 of the block's share of S for the A B pass, 2^-10 of that for the two lo
  passes) and promoted into the accumulator with one rounded add (2^-24 S_ij each, 3 ceil(K / 32) of them), so
  tau = 3 2^-20 + 2^-17 (1 + 2^-9) + 3 ceil(K / 32) 2^-24.

The aggregate bars of the other GEMM tests stay on the normalised error max |C - ref| / S: tf32 below 2e-5, 3xTF32
below 2e-6 sqrt(max(1, K / 256)) and at least 20 times below one truncating tf32 pass on the same operands.

Column sums (want_colsum) are checked against the stored C: |colsum_j - sum_i C_ij| <= 2e-5 sum_i |C_ij|."""
import math
import os

import pytest
import torch

import enhancing_transformers_b200 as etb

pytestmark = pytest.mark.gpu
ops = etb.ops
CAPPED_CTAS = 2
KINDS = ["tf32_bn64", "tf32_bn128", "3xtf32"]
LAYOUTS = [(0, 0), (0, 1), (1, 1), (1, 0)]


@pytest.fixture(autouse=True)
def _restore_sm_limit():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    torch.manual_seed(0)
    yield
    ops.set_sm_limit(int(os.environ.get("B200VQ_SM_LIMIT", "0") or 0))


def tf32_rn(t):
    i = t.contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1fff).view(torch.float32)


def tile_cols(kind):
    return 128 if kind == "tf32_bn128" else 64       # the 3xTF32 product always runs on 64-column tiles


def tiles(kind, M, N, splits=1):
    return -(-M // 128) * -(-N // tile_cols(kind)) * splits


def tau(kind, K):
    if kind == "3xtf32":
        return 3 * 2.0 ** -20 + 2.0 ** -17 * (1 + 2.0 ** -9) + 3 * math.ceil(K / 32) * 2.0 ** -24
    return K * 2.0 ** -22


def logical_operands(kind, M, N, K):
    """A [M, K] and B [N, K] with power-of-two row scales; rounded to tf32 for the tf32 kinds"""
    a = torch.randn(M, K, device="cuda") * 2.0 ** torch.randint(-8, 9, (M, 1), device="cuda")
    b = torch.randn(N, K, device="cuda") * 2.0 ** torch.randint(-8, 9, (N, 1), device="cuda")
    return (a, b) if kind == "3xtf32" else (tf32_rn(a), tf32_rn(b))


def stored(x, major):
    """the operand as the kernel reads it: [rows, K] for major 0, a transposed contiguous copy [K, rows] for major 1"""
    return x if major == 0 else x.t().contiguous()


def gemm(kind, a, b, M, N, K, **kw):
    """one product on `kind` from the stored operands a, b (the 3xTF32 residues are split from the same tensors)"""
    if kind == "3xtf32":
        return ops.gemm(a, b, M, N, K, a_lo=ops.split_tf32_lo(a), b_lo=ops.split_tf32_lo(b), **kw)
    return ops.gemm(a, b, M, N, K, bn=tile_cols(kind), **kw)


def full_and_capped(fn):
    """fn() on the full grid and on CAPPED_CTAS CTAs"""
    ops.set_sm_limit(0)
    full = fn()
    ops.set_sm_limit(CAPPED_CTAS)
    capped = fn()
    ops.set_sm_limit(0)
    torch.cuda.synchronize()
    return full, capped


def assert_same_bits(x, y, what):
    """bit-for-bit equality, with where the differences are if there are any"""
    if x.view(torch.int32).equal(y.view(torch.int32)):
        return
    d = (x.view(torch.int32) != y.view(torch.int32)).reshape(-1, x.shape[-1]).nonzero()
    rows, cols = d[:, 0], d[:, 1]
    raise AssertionError(f"{what}: {len(d)} elements differ; first at {tuple(d[0].tolist())}; row blocks "
                         f"{sorted(set((rows // 128).tolist()))[:16]}, 16-row groups {sorted(set((rows // 16).tolist()))[:16]}, "
                         f"n8 tiles {sorted(set((cols // 8).tolist()))[:16]}")


def assert_within(c, ref, bound, what):
    err = (c.double() - ref).abs()
    bad = ~(err <= bound)                               # NaN fails
    if bad.any():
        d = bad.nonzero()
        i, j = d[0].tolist()
        raise AssertionError(f"{what}: {len(d)} elements outside the bound; first at ({i}, {j}): C {c[i, j].item():.9g}, "
                             f"fp64 {ref[i, j].item():.9g}, |err| {err[i, j].item():.3g} > {bound[i, j].item():.3g}; rows "
                             f"{sorted(set(d[:, 0].tolist()))[:16]}, n8 tiles {sorted(set((d[:, 1] // 8).tolist()))[:16]}")


def normalised_error(c, pre, S):
    return ((c.double() - pre).abs() / S.clamp_min(1e-300)).max().item()


def assert_colsum(cs, c, what):
    err = (cs.double() - c.double().sum(0)).abs()
    bound = 2e-5 * c.double().abs().sum(0)
    assert (err <= bound).all(), f"{what}: column sums off in columns {(err > bound).nonzero().flatten()[:16].tolist()}"


# ------------------------------------------------------------------------------------------ epilogue forms
def epilogue_inputs(form, M, N, mod):
    kw = {}
    if form.startswith("bias"):
        kw["bias"] = torch.randn(N, device="cuda")
    if form == "bias_tanh":
        kw["act"] = 1
    elif form == "bias_residual":
        kw["res"] = torch.randn(M, N, device="cuda")
    elif form == "bias_table":
        kw["res"], kw["res_row_mod"] = torch.randn(mod, N, device="cuda"), mod
    elif form == "tanh_grad":
        kw["aux"], kw["want_colsum"] = torch.tanh(torch.randn(M, N, device="cuda")), True
    return kw


def reference_and_bound(kw, pre, S, t):
    """fp64 epilogue (header order: + bias, tanh, * (1 - aux^2), + residual / table row) on the exact product pre,
    and the per-element bound tau S g + eps"""
    y = pre + kw["bias"].double() if "bias" in kw else pre
    g, eps = 1.0, (2.0 ** -23 * y.abs() if "bias" in kw else 0.0)
    if kw.get("act") == 1:
        ref = torch.tanh(y)
        eps = eps + 6e-7
    elif "aux" in kw:
        f = 1 - kw["aux"].double() ** 2
        ref = y * f
        g, eps = f.abs(), 2.0 ** -23 * (y.abs() + ref.abs())      # 1 - a^2 to 2^-24 absolute, then one product rounding
    elif "res" in kw:
        r = kw["res"].double()
        if kw.get("res_row_mod"):
            r = r[torch.arange(pre.shape[0], device="cuda") % kw["res_row_mod"]]
        ref = y + r
        eps = eps + 2.0 ** -23 * ref.abs()
    else:
        ref = y
    return ref, t * S * g + eps


# (form, (a_major, b_major), M, N, K, table rows): the layouts each form takes in functional.py.  The ragged cases
# leave a 104-row last row block (M 1000), an 8-column last column block (N 648) and an 8-deep last k-block (K 200);
# the others are the default path's patch embedding, pre_quant, post_quant and to_pixel at 2 images.
CASES = [
    ("plain", (0, 0), 1000, 648, 200, 0),
    ("plain", (0, 1), 992, 608, 200, 0),             # dgrad; MN-major B needs N in whole 32-element atoms
    ("plain", (0, 1), 2048, 192, 768, 0),            # to_pixel
    ("bias", (0, 0), 1000, 648, 200, 0),
    ("bias", (0, 0), 2048, 32, 768, 0),              # pre_quant
    ("bias_tanh", (0, 0), 1000, 648, 200, 0),
    ("bias_residual", (0, 0), 1000, 648, 200, 0),
    ("bias_table", (0, 0), 1000, 648, 200, 384),     # 384 does not divide 1000
    ("bias_table", (0, 0), 2048, 768, 192, 1024),    # patch embedding
    ("bias_table", (0, 0), 2048, 768, 32, 1024),     # post_quant
    ("tanh_grad", (0, 1), 992, 608, 200, 0),         # fc1's dgrad with its bias gradient
]
CASE_IDS = [f"{f}-{am}{bm}-{M}x{N}x{K}" + (f"-mod{mod}" if mod else "") for f, (am, bm), M, N, K, mod in CASES]


def run_case(kind, case):
    """the case's operands and epilogue inputs, and fn(kind, **extra) running it on a kind"""
    form, (am, bm), M, N, K, mod = case
    a, b = logical_operands(kind, M, N, K)
    kw = epilogue_inputs(form, M, N, mod)
    sa, sb = stored(a, am), stored(b, bm)
    return a, b, kw, lambda k=kind, **extra: gemm(k, sa, sb, M, N, K, a_major=am, b_major=bm, **kw, **extra)


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
@pytest.mark.parametrize("kind", KINDS)
def test_epilogue_form_capped_grid_bits_and_fp64(kind, case):
    form, _, M, N, K, _ = case
    assert tiles(kind, M, N) >= 8 * CAPPED_CTAS
    a, b, kw, fn = run_case(kind, case)
    full, capped = full_and_capped(fn)
    if kw.get("want_colsum"):
        assert_same_bits(full[0], capped[0], "C, full vs capped grid")
        assert_same_bits(full[1], capped[1], "column sums, full vs capped grid")
        c, cs = capped
        assert_colsum(cs, c, form)
    else:
        assert_same_bits(full, capped, "C, full vs capped grid")
        c = capped
    A, B = a.double(), b.double()
    pre, S = A @ B.t(), A.abs() @ B.abs().t()
    ref, bound = reference_and_bound(kw, pre, S, tau(kind, K))
    assert_within(c, ref, bound, f"{kind} {form}")


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_tf32_tile_widths_give_identical_bits(case):
    _, _, kw, fn = run_case("tf32_bn64", case)
    r64, r128 = fn("tf32_bn64"), fn("tf32_bn128")
    if kw.get("want_colsum"):
        assert_same_bits(r64[0], r128[0], "C, BN 64 vs BN 128")
        assert_same_bits(r64[1], r128[1], "column sums, BN 64 vs BN 128")
    else:
        assert_same_bits(r64, r128, "C, BN 64 vs BN 128")


@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
@pytest.mark.parametrize("kind", ["tf32_bn64", "tf32_bn128"])
def test_tf32_round_out_is_tf32_rn_of_the_output(kind, case):
    _, _, kw, fn = run_case(kind, case)
    c, cr = fn(), fn(round_out=True)
    if kw.get("want_colsum"):
        assert_same_bits(cr[0], tf32_rn(c[0]), "round_out vs tf32_rn")
        assert_colsum(cr[1], cr[0], "column sums of the rounded output")
    else:
        assert_same_bits(cr, tf32_rn(c), "round_out vs tf32_rn")


# ------------------------------------------------------------------------------------------ operand layouts
LM, LN, LK = 992, 608, 200       # MN-major operands need M and N in whole 32-element atoms; K stays ragged


@pytest.mark.parametrize("kind", KINDS)
def test_all_four_layouts_give_identical_bits(kind):
    a, b = logical_operands(kind, LM, LN, LK)
    out = {lay: gemm(kind, stored(a, lay[0]), stored(b, lay[1]), LM, LN, LK, a_major=lay[0], b_major=lay[1]) for lay in LAYOUTS}
    for lay in LAYOUTS[1:]:
        assert_same_bits(out[lay], out[(0, 0)], f"layout {lay} vs (0, 0)")
    A, B = a.double(), b.double()
    pre, S = A @ B.t(), A.abs() @ B.abs().t()
    assert_within(out[(1, 0)], pre, tau(kind, LK) * S, f"{kind} layout (1, 0)")


def wide(x, pad):
    """x in the leading columns of a buffer `pad` columns wider, the padding NaN: the kernel must never read it"""
    buf = torch.full((x.shape[0], x.shape[1] + pad), float("nan"), device="cuda")
    buf[:, :x.shape[1]] = x
    return buf


@pytest.mark.parametrize("layout", LAYOUTS, ids=[f"{am}{bm}" for am, bm in LAYOUTS])
@pytest.mark.parametrize("kind", KINDS)
def test_strided_operands_give_identical_bits(kind, layout):
    am, bm = layout
    a, b = logical_operands(kind, LM, LN, LK)
    sa, sb = stored(a, am), stored(b, bm)
    pa, pb = (12 if am == 0 else 32), (12 if bm == 0 else 32)      # lda / ldb = K + 12 (K-major), rows + 32 (MN-major)
    wa, wb = wide(sa, pa), wide(sb, pb)
    contiguous = gemm(kind, sa, sb, LM, LN, LK, a_major=am, b_major=bm)
    strided = gemm(kind, wa, wb, LM, LN, LK, a_major=am, b_major=bm, lda=sa.shape[1] + pa, ldb=sb.shape[1] + pb)
    assert_same_bits(strided, contiguous, f"lda {sa.shape[1] + pa} / ldb {sb.shape[1] + pb} vs contiguous")


# ------------------------------------------------------------------------------------------ split-K wgrad
@pytest.mark.parametrize("rows,cols,K", [(992, 608, 224), (768, 192, 672)], ids=["ragged", "patch_embed_wgrad"])
@pytest.mark.parametrize("kind", KINDS)
def test_split_k_slices_and_reduce(kind, rows, cols, K):
    """dW[rows, cols] = dY^T X over 3 K-slices (both operands MN-major, as _wgrad runs it)"""
    splits = 3
    assert tiles(kind, rows, cols, splits) >= 8 * CAPPED_CTAS
    dyT, xT = logical_operands(kind, rows, cols, splits * K)                # dY^T [rows, 3K], X^T [cols, 3K]
    A, B = dyT.t().contiguous(), xT.t().contiguous()                        # stored [3K, rows], [3K, cols]
    full, part = full_and_capped(lambda: gemm(kind, A, B, rows, cols, K, a_major=1, b_major=1, splits=splits))
    assert part.shape == (splits, rows, cols)
    assert_same_bits(full, part, "split-K partials, full vs capped grid")
    Ad, Bd = dyT.double(), xT.double()
    for z in range(splits):
        alone = gemm(kind, A[z * K:(z + 1) * K].contiguous(), B[z * K:(z + 1) * K].contiguous(), rows, cols, K, a_major=1, b_major=1)
        assert_same_bits(part[z], alone, f"split {z} vs the same slice alone")
        az, bz = Ad[:, z * K:(z + 1) * K], Bd[:, z * K:(z + 1) * K]
        assert_within(part[z], az @ bz.t(), tau(kind, K) * (az.abs() @ bz.abs().t()), f"{kind} split {z}")
    c = ops.splitk_reduce(part)
    pre, S = Ad @ Bd.t(), Ad.abs() @ Bd.abs().t()
    assert_within(c, pre, (tau(kind, K) + splits * 2.0 ** -24) * S, f"{kind} reduced")    # + the fp32 sum of the slices


# ------------------------------------------------------------------------------------------ aggregate grades
@pytest.mark.parametrize("kind", KINDS)
def test_normalised_error_grades(kind):
    M, N, K = 1000, 648, 200
    a, b = logical_operands(kind, M, N, K)
    A, B = a.double(), b.double()
    pre, S = A @ B.t(), A.abs() @ B.abs().t()
    e = normalised_error(gemm(kind, a, b, M, N, K), pre, S)
    if kind != "3xtf32":
        assert e < 2e-5, e
        return
    e1 = normalised_error(ops.gemm(a, b, M, N, K), pre, S)                  # one pass: the tensor core truncates
    assert e < 2e-6 * max(1.0, (K / 256) ** 0.5), e
    assert e1 > 20 * e, (e1, e)
