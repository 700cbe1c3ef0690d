"""The row-wise kernels of csrc/rowwise.cu (LayerNorm, colsum, splitk_reduce, the operand conversions, grad_scale, the
re-layouts), and NaN through every tf32 round_out producer, element by element.

Grid sizes.  Every size that depends on the grid is derived from the device's SM count with rowwise.cu's formulas:
the LayerNorm forward runs one warp per row on min(ceil(32 M / 256), 8 SMs) CTAs of 8 warps, so one grid pass covers
64 SMs rows; the backward runs on min(2 SMs, ceil(M / 8)) CTAs, one pass of 16 SMs rows, and leaves that many partial
sums (nparts); colsum runs splits = clamp(ceil(8 SMs / ceil(N / 128)), <= 64, <= ceil(M / 8)) row groups of stride
8 splits; grad_scale's first stage covers min(8 SMs, 1056) * 1024 elements per pass.

Exact checks (no tolerance):
- round_tf32, split_tf32_lo and to_half over all 2^32 fp32 bit patterns, in 2^25-element chunks: round_tf32 is
  (u + 0x1000) & 0xFFFFE000 for every non-NaN u (round to nearest, ties away; FLT_MAX's neighbourhood rounds to inf)
  and (u | 0x00400000) & 0xFFFFE000 for a NaN; split_tf32_lo is x - (x & 0xFFFFE000) as torch computes it;
  to_half is x.clamp(+-65504).half() (half subnormals and ties included), NaN giving NaN.
- NaN through every round_out producer (LayerNorm forward and backward, patchify, the tf32 GEMM, time_mix, sqrelu and
  its derivative): the rows that hold a NaN come out NaN, every other row is bit-identical to a NaN-free run.
- LayerNorm rows are independent: rows [i0, i1), launched alone through a slice that starts at an odd row, give the
  bits of the same rows of a launch whose forward loops 4 grid passes and whose backward loops more than 4.
- LayerNorm forms: mean / rstd identical across the y, round_out and y16 forms; y16 = y.clamp(+-65504).half();
  round_out y = tf32_rn(y).  Backward: dx, dgamma and dbeta identical with and without column sums (2 or 3
  accumulators) and the fp16 copy; dx16 = (dx * S).clamp(+-65504).half() of the unrounded dx; round_out dx =
  tf32_rn(dx); fp16 dy with dy_scale = the fp32 path fed dyh.float() * (1 / S), at D % 8 == 0 (16-byte loads staged
  through shared memory) and D % 8 == 4 (8-byte loads).  Two runs give the same dgamma, dbeta, dxsum and colsum.
- splitk_reduce is torch's sequential fp32 sum over the splits times alpha; patchify / unpatchify / add_rows_mod are
  torch's reshape / permute / indexing.
- grad_scale gives S = 2^clamp(t - ceil(log2 max|g|), -100, 100) exactly (max|g| * S in (2^(t-1), 2^t]), and {1, 1}
  when max|g| is 0, inf or NaN.

fp64 checks, per element |out - ref| <= bound (NaN fails), u = 2^-24.  A row sum in these kernels adds a float4's four
values as (a + b) + (c + d), adds k = ceil(D / 128) such sums into the lane's running sum (the first add is exact),
folds the 32 lanes in L = ceil(log2 min(D / 4, 32)) butterfly levels that add two non-zero values (lanes past D / 4
hold 0) and divides by D: h = k + L + 2 roundings on the longest path, so a computed mean is off by at most
h u mean|term|.  With A = mean|x|, sigma^2 the exact variance and V = sigma^2 + eps:
- mean: |mu_k - mu| <= dmu = h u A.
- rstd: (x - mu_k)^2 carries 3 roundings and its sum h, and sum (x - mu_k)^2 / D = sigma^2 + (mu - mu_k)^2, so
  V_k / V - 1 <= eps_V = ((h + 3) u (sigma^2 + dmu^2) + dmu^2) / V + u (the + eps); rsqrtf is within 2 ulp (4 u), so
  |rstd_k / rstd - 1| <= eps_r = eps_V / 2 (1 + eps_V) + 4 u (1 + eps_V).
- y = (x - mu_k) rstd_k gamma + beta: |gamma| rstd (1 + eps_r) dmu (the mean) + |gamma xhat| eps_r (the rsqrt) +
  3 u of the product and u of the sum.
- dx, isolated from the forward by evaluating the fp64 formula on the kernel's own mean and rstd: h = (x - mu) rstd
  (2 roundings), t = dy gamma (1), m1 = mean(t), m2 = mean(t h) (h + 1 and h + 4 roundings of mean|t| and mean|t h|),
  w = t - m1 - h m2 (3), dx = rstd w + dres (2).
- dgamma / dbeta / dxsum: a warp adds ceil(M / (8 nparts)) rows, the CTA adds its 8 warps, ln_param_reduce adds
  ceil(nparts / 16) partials in each of two chains, the two chains and the 8 warps: hp = ceil(M / (8 nparts)) + 8 +
  ceil(nparts / 16) + 9, bound hp u sum|term| (+ 3 u for dgamma's rounded dy h).  dxsum is checked against the sum of
  the stored dx.
- colsum: a thread adds at most ceil(M / stride) rows in four chains joined by 3 adds, then 8 row lanes and the splits
  partials: (ceil(M / stride) + 11 + splits) u sum|x|.
The rows are N(0, 1) scaled by 2^r, r in [-8, 8], with eps-dominated rows (sigma 1e-4), offset rows (mean / sigma
256, where a one-pass variance E[x^2] - mu^2 misses the bound by far more than 10 times: asserted on the inputs),
all-zero rows (y is beta bit for bit), constant rows and one-spike rows; gamma has zeros and negatives."""
import math

import pytest
import torch

import enhancing_transformers_b200 as etb

pytestmark = pytest.mark.gpu
ops = etb.ops
H = torch.float16
U = 2.0 ** -24
EPS = torch.tensor(1e-5, dtype=torch.float32).item()          # the kernel's kLnEps, as an fp64 number
GRADES = {}                                                    # check -> largest |err| / bound seen (reported with -s)


@pytest.fixture(autouse=True)
def _need_cuda():
    assert torch.cuda.is_available(), "-m gpu tests need a CUDA device"
    torch.manual_seed(0)


@pytest.fixture(scope="module", autouse=True)
def _report_grades():
    yield
    for k in sorted(GRADES):
        print(f"\n  grade {k}: {GRADES[k]:.3g}", end="")
    for k, v in NAN_NOTES.items():
        print(f"\n  {k}: bits {[hex(b & 0xFFFFFFFF) for b in v]}", end="")
    print(f"\n  peak device memory allocated: {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def fwd_rows_per_pass():
    return 64 * sms()


def bwd_rows_per_pass():
    return 16 * sms()


def bwd_parts(M):
    return min(2 * sms(), -(-M // 8))


def colsum_splits(M, N):
    colblocks = -(-(N // 4) // 32)
    return max(1, min(-(-8 * sms() // colblocks), 64, -(-M // 8)))


def absmax_pass():
    return min(8 * sms(), 1056) * 1024


def tf32_rn(t):
    """round_tf32's rule on the bits: ties away from zero; a NaN keeps its sign and gets the quiet bit"""
    i = t.contiguous().view(torch.int32)
    nan = (i & 0x7FFFFFFF) > 0x7F800000
    return (torch.where(nan, i | 0x00400000, i + 0x1000) & ~0x1FFF).view(torch.float32)


def from_bits(*patterns):
    return torch.tensor([p - (1 << 32) if p >= 1 << 31 else p for p in patterns], dtype=torch.int32, device="cuda").view(torch.float32)


def bits(t):
    return t.contiguous().view(torch.int16 if t.dtype == H else torch.int32)


def first_diff(d, shape):
    """'flat index i (row r)' of the first True of the flat mask d, and how many there are"""
    idx = d.nonzero().flatten()
    i = idx[0].item()
    cols = shape[-1] if len(shape) > 1 else max(1, d.numel())
    return i, f"{len(idx)} elements; first at flat index {i} (row {i // cols}, column {i % cols}); rows " \
              f"{sorted(set((idx // cols).tolist()))[:12]}"


def assert_same_bits(x, y, what):
    assert x.shape == y.shape and x.dtype == y.dtype, f"{what}: {x.shape} {x.dtype} vs {y.shape} {y.dtype}"
    bx, by = bits(x).flatten(), bits(y).flatten()
    if bx.equal(by):
        return
    i, where = first_diff(bx != by, x.shape)
    raise AssertionError(f"{what}: differ at {where}: {x.flatten()[i].item()!r} vs {y.flatten()[i].item()!r}")


def assert_same_or_both_nan(x, y, what):
    """bit-identical where y is not NaN, NaN exactly where y is NaN"""
    nx, ny = torch.isnan(x).flatten(), torch.isnan(y).flatten()
    bx, by = bits(x).flatten(), bits(y).flatten()
    if not nx.equal(ny):
        i, where = first_diff(nx != ny, x.shape)
        raise AssertionError(f"{what}: NaN-ness differs at {where}: got bits {bx[i].item() & 0xFFFFFFFF:#x}, "
                             f"want {by[i].item() & 0xFFFFFFFF:#x} (input {i})")
    d = (bx != by) & ~ny
    if d.any():
        i, where = first_diff(d, x.shape)
        raise AssertionError(f"{what}: differ at {where}: bits {bx[i].item() & 0xFFFFFFFF:#x} vs {by[i].item() & 0xFFFFFFFF:#x}")


def assert_within(out, ref, bound, what):
    """|out - ref| <= bound per element (NaN fails); records the largest |err| / bound under `what`"""
    err = (out.double() - ref).abs()
    bound = bound.expand_as(err)
    bad = ~(err <= bound)
    if bad.any():
        i, where = first_diff(bad.flatten(), err.shape)
        o, r, e, b = (t.flatten()[i].item() for t in (out, ref, err, bound))
        raise AssertionError(f"{what}: outside the bound at {where}: got {o:.9g}, fp64 {r:.9g}, |err| {e:.3g} > {b:.3g}")
    g = (err / bound.clamp_min(1e-300)).max().item() if err.numel() else 0.0
    GRADES[what] = max(GRADES.get(what, 0.0), g)


# ------------------------------------------------------------------------------ every fp32 bit pattern
CHUNK = 1 << 25


def all_fp32_chunks():
    """every fp32 bit pattern once, as int32 tensors of CHUNK patterns"""
    base = torch.arange(CHUNK, dtype=torch.int32, device="cuda")
    for c in range(1 << 32 >> 25):
        off = c << 25
        yield base | (off - (1 << 32) if off >= 1 << 31 else off)


def test_round_tf32_every_bit_pattern():
    for u in all_fp32_chunks():
        got = ops.round_tf32(u.view(torch.float32)).view(torch.int32).long() & 0xFFFFFFFF
        w = u.long() & 0xFFFFFFFF
        nan = (w & 0x7FFFFFFF) > 0x7F800000
        want = torch.where(nan, w | 0x00400000, w + 0x1000) & 0xFFFFE000
        if not got.equal(want):
            i = (got != want).nonzero()[0].item()
            raise AssertionError(f"round_tf32({w[i].item():#010x}) = {got[i].item():#010x}, want {want[i].item():#010x}; "
                                 f"{int((got != want).sum())} patterns of this chunk differ")


def test_split_tf32_lo_every_bit_pattern():
    for u in all_fp32_chunks():
        x = u.view(torch.float32)
        assert_same_or_both_nan(ops.split_tf32_lo(x), x - (u & ~0x1FFF).view(torch.float32),
                                f"split_tf32_lo, patterns {u[0].item() & 0xFFFFFFFF:#010x}..")


def test_to_half_every_bit_pattern():
    for u in all_fp32_chunks():
        x = u.view(torch.float32)
        assert_same_or_both_nan(ops.to_half(x), x.clamp(-65504, 65504).half(), f"to_half, patterns {u[0].item() & 0xFFFFFFFF:#010x}..")


def test_round_tf32_keeps_nan_and_its_sign():
    x = from_bits(0x7FFFFFFF, 0xFFFFFFFF, 0x7F800001, 0xFF800FFF, 0x7FC00000, 0x7FBFFFFF, 0x7F800000, 0xFF800000)
    r = ops.round_tf32(x)
    assert torch.isnan(r[:6]).all(), [hex(v & 0xFFFFFFFF) for v in bits(r).tolist()]
    assert ((bits(r) & 0x1FFF) == 0).all()                          # a tf32 value: the tensor core keeps it whole
    assert ((bits(r) < 0) == (bits(x) < 0)).all()
    assert r[6].item() == math.inf and r[7].item() == -math.inf
    made = torch.tensor([math.inf] * 4, device="cuda")
    made = made - made                                          # NaNs made on the device
    assert torch.isnan(ops.round_tf32(made)).all()


# ------------------------------------------------------------------------------ NaN through round_out producers
NAN_BITS = 0x7FFFFFFF                                           # the NaN fp32 arithmetic on the GPU produces
NAN_NOTES = {}


def plant_nan_rows(x, rows):
    """x with the whole of `rows` set to 0x7FFFFFFF"""
    xn = x.clone()
    xn.view(torch.int32)[rows] = NAN_BITS
    return xn


def check_nan_rows(clean, planted, rows, what, cols=None):
    """rows (and, given a column mask, only those columns of them) NaN; everything else bit-identical to `clean`"""
    mask = torch.zeros(planted.shape[0], dtype=torch.bool, device="cuda")
    mask[rows] = True
    hit = planted[mask] if cols is None else planted[mask][:, cols]
    assert torch.isnan(hit).all(), (
        f"{what}: the NaN rows hold non-NaN values, e.g. bits {sorted(set((bits(hit).flatten() & 0xFFFFFFFF).tolist()))[:4]}")
    assert_same_bits(planted[~mask], clean[~mask], f"{what}: rows without NaN")
    if cols is not None:
        assert_same_bits(planted[mask][:, ~cols], clean[mask][:, ~cols], f"{what}: the rest of the NaN rows")


def producer_layernorm_fwd():
    M, D = 300, 260
    x, g, b = torch.randn(M, D, device="cuda"), torch.randn(D, device="cuda"), torch.randn(D, device="cuda")
    rows = [0, 77, M - 1]
    return ops.layernorm_fwd(x, g, b, True)[0], ops.layernorm_fwd(plant_nan_rows(x, rows), g, b, True)[0], rows


def producer_layernorm_bwd():
    M, D = 300, 516
    x, g = torch.randn(M, D, device="cuda"), torch.randn(D, device="cuda")
    _, mean, rstd = ops.layernorm_fwd(x, g, torch.zeros(D, device="cuda"), False)
    dy, dres = torch.randn(M, D, device="cuda"), torch.randn(M, D, device="cuda")
    rows = [5, 150]
    dyn = dy.clone()
    dyn.view(torch.int32)[rows, 3] = NAN_BITS                   # one element: m1 and m2 spread it over the row
    run = lambda d: ops.layernorm_bwd(d, x, mean, rstd, g, dres, round_out=True)[0]
    return run(dy), run(dyn), rows


def producer_patchify():
    B, C, Hh, W, p = 2, 3, 32, 48, (8, 4)
    img = torch.randn(B, C, Hh, W, device="cuda")
    imgn = img.clone()
    imgn.view(torch.int32)[1, 2, 9, :4] = NAN_BITS              # image row 9 of batch 1, columns 0..3: patch (1, 0)
    rows = [(1 * (Hh // p[0]) + 9 // p[0]) * (W // p[1]) + 0]     # patch (9 // ph, 0) of image 1
    first = (2 * p[0] + 9 % p[0]) * p[1]                          # its (c 2, patch row 9 % ph) piece
    cols = torch.arange(C * p[0] * p[1], device="cuda")
    return ops.patchify(img, p, True), ops.patchify(imgn, p, True), rows, (cols >= first) & (cols < first + p[1])


def producer_gemm_tf32():
    M, N, K = 256, 192, 96
    a, b = tf32_rn(torch.randn(M, K, device="cuda")), tf32_rn(torch.randn(N, K, device="cuda"))
    rows = [3, 200]
    an = plant_nan_rows(a, rows)
    raw = ops.gemm(an, b, M, N, K)
    NAN_NOTES["tf32 GEMM output for a NaN row of A"] = sorted(set((bits(raw[rows]).flatten() & 0xFFFFFFFF).tolist()))
    return ops.gemm(a, b, M, N, K, round_out=True), ops.gemm(an, b, M, N, K, round_out=True), rows


def producer_time_mix():
    B, T, C = 3, 20, 96
    x, w = torch.randn(B * T, C, device="cuda"), torch.rand(C, device="cuda")
    rows = [T - 1, 3 * T - 1]                                   # last step of a sequence: shift(x) takes it nowhere
    return ops.time_mix_fwd(x, w, T, True), ops.time_mix_fwd(plant_nan_rows(x, rows), w, T, True), rows


def producer_sqrelu(grad):
    x = torch.randn(64, 128, device="cuda")
    g = torch.randn_like(x) if grad else None
    rows = [1, 40]
    return ops.sqrelu(x, g, round_out=True), ops.sqrelu(plant_nan_rows(x, rows), g, round_out=True), rows


PRODUCERS = {
    "layernorm_fwd": producer_layernorm_fwd, "layernorm_bwd": producer_layernorm_bwd, "patchify": producer_patchify,
    "gemm_tf32": producer_gemm_tf32, "time_mix_fwd": producer_time_mix, "sqrelu": lambda: producer_sqrelu(False),
    "sqrelu_grad": lambda: producer_sqrelu(True),
}


@pytest.mark.parametrize("producer", list(PRODUCERS))
def test_round_out_keeps_nan(producer):
    clean, planted, rows, *cols = PRODUCERS[producer]()
    check_nan_rows(clean, planted, rows, producer, *cols)


def test_sqrelu_follows_torch_on_nan_inf_and_signed_zero():
    x = torch.randn(32, 64, device="cuda")
    x.view(-1)[:8] = from_bits(0x7FFFFFFF, 0xFFFFFFFF, 0x7FC00000, 0x80000000, 0x00000000, 0x7F800000, 0xFF800000, 0x00000001)
    g = torch.randn_like(x)
    assert_same_or_both_nan(ops.sqrelu(x), torch.square(torch.relu(x)), "sqrelu vs torch.square(torch.relu(x))")
    xr = x.clone().requires_grad_(True)
    torch.square(torch.relu(xr)).backward(g)
    d = ops.sqrelu(x, g)
    assert torch.isnan(d).equal(torch.isnan(xr.grad)), "sqrelu derivative: NaN positions differ from torch"
    keep = ~torch.isnan(d)
    assert torch.equal(d[keep], xr.grad[keep]), "sqrelu derivative differs from torch's"    # -0 == +0 here


# ------------------------------------------------------------------------------ LayerNorm: inputs and bounds
def ln_inputs(M, D, seed=0):
    """rows N(0, 1) 2^r plus special rows by row % 8: 1 eps-dominated, 2 offset (mean / sigma 256), 3 zero, 4 constant,
    5 one spike; gamma with zeros (every 7th) and negatives"""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    sigma = torch.exp2(torch.randint(-8, 9, (M, 1), device="cuda", generator=gen).double())
    kind = (torch.arange(M, device="cuda") % 8).view(M, 1)
    sigma = torch.where(kind == 1, torch.full_like(sigma, 1e-4), sigma)
    z = torch.randn(M, D, device="cuda", generator=gen, dtype=torch.float64)
    x = z * sigma + torch.where(kind == 2, 256 * sigma, torch.zeros_like(sigma))
    x = torch.where(kind == 3, torch.zeros_like(x), x)
    x = torch.where(kind == 4, (z[:, :1] * sigma).expand(M, D), x)
    spike = torch.zeros(M, D, dtype=torch.bool, device="cuda")
    spike[torch.arange(M, device="cuda"), (torch.arange(M, device="cuda") * 7) % D] = True
    x = torch.where(kind == 5, torch.where(spike, 2.0 ** 10 * sigma, z * sigma * 2.0 ** -10), x)
    gamma = torch.randn(D, device="cuda", generator=gen)
    gamma[::7] = 0
    beta = torch.randn(D, device="cuda", generator=gen)
    return x.float(), gamma, beta


def sum_depth(D):
    nv = D // 4
    return -(-nv // 32) + math.ceil(math.log2(min(nv, 32))) + 2


def row_chunks(M, rows=4096):
    return [slice(i, min(M, i + rows)) for i in range(0, M, rows)]


def check_ln_forward(x, gamma, beta, y, mean, rstd, tag):
    M, D = x.shape
    h = sum_depth(D)
    G, Bt = gamma.double(), beta.double()
    for s in row_chunks(M):
        X = x[s].double()
        mu = X.mean(1, keepdim=True)
        var = ((X - mu) ** 2).mean(1, keepdim=True)
        V = var + EPS
        r = V.rsqrt()
        dmu = h * U * X.abs().mean(1, keepdim=True)
        eps_v = ((h + 3) * U * (var + dmu ** 2) + dmu ** 2) / V + U
        eps_r = 0.5 * eps_v * (1 + eps_v) + 4 * U * (1 + eps_v)
        assert_within(mean[s].view(-1, 1), mu, dmu * (1 + 1e-6), f"LN forward mean {tag}")
        assert_within(rstd[s].view(-1, 1), r, eps_r * r * (1 + 1e-6), f"LN forward rstd {tag}")
        xh = (X - mu) * r
        yref = xh * G + Bt
        mean_term = G.abs() * r * (1 + eps_r) * dmu
        rsqrt_term = (G * xh).abs() * eps_r
        prod = (G * xh).abs() * (1 + eps_r) + mean_term
        b = mean_term + rsqrt_term + 3 * U * prod
        b = (b + U * (yref.abs() + b)) * (1 + 1e-6)
        assert_within(y[s], yref, b, f"LN forward y {tag}")
        if tag == "fp64":
            # the offset rows are there for a one-pass variance: its fp32 rstd must miss eps_r by far
            off = (torch.arange(s.start, s.stop, device="cuda") % 8 == 2)
            if off.any():
                xf = x[s][off]
                one_pass = (xf * xf).mean(1, keepdim=True) - xf.mean(1, keepdim=True) ** 2
                r1 = (one_pass.clamp_min(0) + EPS).rsqrt().double()
                assert ((r1 - r[off]).abs() / (eps_r[off] * r[off])).max().item() >= 10
    zero = (torch.arange(M, device="cuda") % 8 == 3)
    if zero.any():
        assert_same_bits(y[zero], beta.expand(int(zero.sum()), D), "LN forward: y of an all-zero row is beta")


def check_ln_backward(x, gamma, dy, dres, mean, rstd, dx, dgamma, dbeta, dxsum, tag):
    M, D = x.shape
    h = sum_depth(D)
    nparts = bwd_parts(M)
    hp = -(-M // (8 * nparts)) + 8 + -(-nparts // 16) + 9
    G = gamma.double()
    sg, sb, sx = (torch.zeros(D, dtype=torch.float64, device="cuda") for _ in range(3))
    ag, ab, ax = (torch.zeros(D, dtype=torch.float64, device="cuda") for _ in range(3))
    for s in row_chunks(M):
        X, DY, DR = x[s].double(), dy[s].double(), dres[s].double()
        mu, r = mean[s].double().view(-1, 1), rstd[s].double().view(-1, 1)
        Hh = (X - mu) * r
        T = DY * G
        m1, m2 = T.mean(1, keepdim=True), (T * Hh).mean(1, keepdim=True)
        W = T - m1 - Hh * m2
        ref = r * W + DR
        b = r * (2 * U * T.abs() + U * m1.abs() + 3 * U * (Hh * m2).abs() + (h + 1) * U * T.abs().mean(1, keepdim=True)
                 + (h + 4) * U * Hh.abs() * (T * Hh).abs().mean(1, keepdim=True) + 2 * U * W.abs())
        b = (b + U * ref.abs()) * (1 + 1e-5)
        assert_within(dx[s], ref, b, f"LN backward dx {tag}")
        sg += (DY * Hh).sum(0); ag += (DY * Hh).abs().sum(0)
        sb += DY.sum(0); ab += DY.abs().sum(0)
        sx += dx[s].double().sum(0); ax += dx[s].double().abs().sum(0)
    assert_within(dgamma, sg, (hp + 3) * U * ag * (1 + 1e-6), f"LN backward dgamma {tag}")
    assert_within(dbeta, sb, hp * U * ab * (1 + 1e-6), f"LN backward dbeta {tag}")
    if dxsum is not None:
        assert_within(dxsum, sx, hp * U * ax * (1 + 1e-6), f"LN backward dxsum {tag}")


LN_DS = [4, 124, 128, 132, 252, 256, 260, 508, 512, 516, 764, 768, 772, 1276, 1280, 1284, 2044, 2048]
LN_MS = ["1", "7", "9", "bwd_pass-1", "bwd_pass+1", "fwd_pass+1"]


def resolve_m(m):
    return {"bwd_pass-1": bwd_rows_per_pass() - 1, "bwd_pass+1": bwd_rows_per_pass() + 1,
            "fwd_pass+1": fwd_rows_per_pass() + 1}.get(m) or int(m)


@pytest.mark.parametrize("D,m", [(D, m) for D in LN_DS for m in LN_MS] + [(768, "65536")])   # 65536: base batch 64
def test_layernorm_fp64(D, m):
    M = resolve_m(m)
    x, gamma, beta = ln_inputs(M, D, seed=D + M)
    y, mean, rstd = ops.layernorm_fwd(x, gamma, beta, False)
    check_ln_forward(x, gamma, beta, y, mean, rstd, "fp64")
    del y
    gen = torch.Generator(device="cuda").manual_seed(7 * D + M)
    dy = torch.randn(M, D, device="cuda", generator=gen) * torch.exp2(torch.randint(-8, 9, (M, 1), device="cuda", generator=gen).float())
    dres = torch.randn(M, D, device="cuda", generator=gen)
    dx, dg, db, dxs = ops.layernorm_bwd(dy, x, mean, rstd, gamma, dres, want_colsum=True)
    check_ln_backward(x, gamma, dy, dres, mean, rstd, dx, dg, db, dxs, "fp64")


# ------------------------------------------------------------------------------ LayerNorm: exact invariants
@pytest.mark.parametrize("D", [260, 1284])
def test_layernorm_rows_are_independent_of_the_launch(D):
    M = 3 * fwd_rows_per_pass() + 37                              # forward: 4 grid passes; backward: 12 and more
    assert M > 2 * fwd_rows_per_pass() and M > 3 * bwd_rows_per_pass()
    x, gamma, beta = ln_inputs(M, D, seed=11)
    dy, dres = torch.randn(M, D, device="cuda"), torch.randn(M, D, device="cuda")
    y, mean, rstd = ops.layernorm_fwd(x, gamma, beta, False)
    dx = ops.layernorm_bwd(dy, x, mean, rstd, gamma, dres)[0]
    i0 = fwd_rows_per_pass() + bwd_rows_per_pass() + 1            # odd, inside the second forward pass
    i1 = i0 + fwd_rows_per_pass() + 2 * bwd_rows_per_pass() + 5   # into the third forward pass
    assert i0 % 2 == 1 and 3 * fwd_rows_per_pass() > i1 > 2 * fwd_rows_per_pass()
    ys, ms, rs = ops.layernorm_fwd(x[i0:i1], gamma, beta, False)
    assert_same_bits(ys, y[i0:i1], "y of rows launched alone")
    assert_same_bits(ms, mean[i0:i1], "mean of rows launched alone")
    assert_same_bits(rs, rstd[i0:i1], "rstd of rows launched alone")
    dxs = ops.layernorm_bwd(dy[i0:i1], x[i0:i1], mean[i0:i1], rstd[i0:i1], gamma, dres[i0:i1])[0]
    assert_same_bits(dxs, dx[i0:i1], "dx of rows launched alone")


@pytest.mark.parametrize("D", [124, 1284, 2048])
def test_layernorm_forward_forms_agree(D):
    M = bwd_rows_per_pass() + 3
    x, gamma, beta = ln_inputs(M, D, seed=3)
    gamma[1::5] = 3e4 * torch.sign(gamma[1::5])                     # |y| past 65504 in many rows
    y, mean, rstd = ops.layernorm_fwd(x, gamma, beta, False)
    yr, mean_r, rstd_r = ops.layernorm_fwd(x, gamma, beta, True)
    yh, mean_h, rstd_h = ops.layernorm_fwd(x, gamma, beta, False, out_half=True)
    assert (y.abs() > 65504).any()
    for m2, r2, form in ((mean_r, rstd_r, "round_out"), (mean_h, rstd_h, "y16")):
        assert_same_bits(m2, mean, f"mean, {form} form")
        assert_same_bits(r2, rstd, f"rstd, {form} form")
    assert_same_bits(yr, tf32_rn(y), "round_out y vs tf32_rn(y)")
    assert_same_bits(yh, y.clamp(-65504, 65504).half(), "y16 vs the saturating half of y")


def ln_bwd_case(M, D, seed):
    x, gamma, beta = ln_inputs(M, D, seed=seed)
    _, mean, rstd = ops.layernorm_fwd(x, gamma, beta, False)
    gen = torch.Generator(device="cuda").manual_seed(seed + 1)
    dy = torch.randn(M, D, device="cuda", generator=gen) * 3
    dres = torch.randn(M, D, device="cuda", generator=gen)
    return x, gamma, mean, rstd, dy, dres


@pytest.mark.parametrize("D", [4, 124, 132, 512, 516, 1276, 1280, 2044, 2048])
def test_layernorm_backward_forms_agree(D):
    M = 2 * bwd_rows_per_pass() + 7
    x, gamma, mean, rstd, dy, dres = ln_bwd_case(M, D, seed=D)
    S = torch.tensor([2.0 ** 12], device="cuda")                  # large enough that some |dx S| pass 65504
    bwd = lambda d, **kw: ops.layernorm_bwd(d, x, mean, rstd, gamma, dres, **kw)
    dx, dg, db = bwd(dy)
    dx_c, dg_c, db_c, dxs = bwd(dy, want_colsum=True)
    dx_h, dg_h, db_h, dx16 = bwd(dy, half_scale=S)
    dx_r, dg_r, db_r, dxs_r, dx16_r = bwd(dy, round_out=True, want_colsum=True, half_scale=S)
    for (a, b_, c), form in (((dx_c, dg_c, db_c), "column sums"), ((dx_h, dg_h, db_h), "fp16 copy")):
        assert_same_bits(a, dx, f"dx with the {form}")
        assert_same_bits(b_, dg, f"dgamma with the {form}")
        assert_same_bits(c, db, f"dbeta with the {form}")
    assert_same_bits(dg_r, dg, "dgamma with round_out")
    assert_same_bits(db_r, db, "dbeta with round_out")
    assert (dx * S).abs().max() > 65504
    assert_same_bits(dx16, (dx * S).clamp(-65504, 65504).half(), "dx16 vs the saturating half of dx S")
    assert_same_bits(dx16_r, dx16, "dx16 with round_out comes from the unrounded dx")
    assert_same_bits(dx_r, tf32_rn(dx), "round_out dx vs tf32_rn(dx)")
    # fp16 dy carrying a gradient scale: read as dyh * (1 / S), the same values as the fp32 path is given
    sc = ops.grad_scale(dy)
    dyh = ops.to_half(dy, sc[0:1])
    dy_rt = dyh.float() * sc[1]
    for kw in ({}, {"want_colsum": True}, {"want_colsum": True, "half_scale": S, "round_out": True}):
        ref, got = bwd(dy_rt, **kw), bwd(dyh, dy_scale=sc[1:2], **kw)
        for i, (a, b_) in enumerate(zip(got, ref)):
            assert_same_bits(a, b_, f"fp16 dy ({'16-byte staged' if D % 8 == 0 else '8-byte'} loads) {sorted(kw)} output {i}")


@pytest.mark.parametrize("D,dy_half", [(768, False), (2048, True), (772, True)])
def test_layernorm_backward_and_colsum_are_deterministic(D, dy_half):
    M = 3 * bwd_rows_per_pass() + 5
    x, gamma, mean, rstd, dy, dres = ln_bwd_case(M, D, seed=5)
    kw = {}
    if dy_half:
        sc = ops.grad_scale(dy)
        dy, kw = ops.to_half(dy, sc[0:1]), {"dy_scale": sc[1:2]}
    a = ops.layernorm_bwd(dy, x, mean, rstd, gamma, dres, want_colsum=True, **kw)
    b = ops.layernorm_bwd(dy, x, mean, rstd, gamma, dres, want_colsum=True, **kw)
    for i, name in enumerate(["dx", "dgamma", "dbeta", "dxsum"]):
        assert_same_bits(a[i], b[i], f"{name}, two runs")
    assert_same_bits(ops.colsum(a[0]), ops.colsum(b[0]), "colsum, two runs")


# ------------------------------------------------------------------------------ colsum
COLSUM_MS = {"3s-1": (3, -1), "3s": (3, 0), "3s+1": (3, 1), "4s-1": (4, -1), "4s+1": (4, 1), "4s+43": (4, 43)}


def resolve_colsum(m, n):
    """M in units of the row stride 8 splits (3 s - 1 leaves the 4-way body unused, 4 s + 1 runs it once plus the
    tail), or a literal; N literal or 'one_split' (+ extra): as many 128-column blocks as 8 SMs, so splits = 1"""
    N = 128 * 8 * sms() + int(n.split("+")[1]) if n.startswith("one_split") else int(n)
    if m in COLSUM_MS:
        k, d = COLSUM_MS[m]
        return k * 8 * colsum_splits(1 << 24, N) + d, N
    return int(m), N


@pytest.mark.parametrize("m,n", [(m, n) for n in ("4", "124", "132", "388") for m in list(COLSUM_MS) + ["5"]]
                         + [("37", "one_split+0"), ("37", "one_split+132"), ("3", "one_split+4")])
def test_colsum_fp64(m, n):
    M, N = resolve_colsum(m, n)
    splits = colsum_splits(M, N)
    assert splits == 1 if n.startswith("one_split") or M < 8 else splits > 1
    x = torch.randn(M, N, device="cuda") * torch.exp2(torch.randint(-8, 9, (M, 1), device="cuda").float())
    cs = ops.colsum(x)
    X = x.double()
    chain = -(-M // (8 * splits))
    assert_within(cs, X.sum(0), (chain + 11 + splits) * U * X.abs().sum(0) * (1 + 1e-6), "colsum")
    assert_same_bits(ops.colsum(x), cs, "colsum, two runs")


# ------------------------------------------------------------------------------ splitk_reduce
@pytest.mark.parametrize("splits", range(1, 9))
def test_splitk_reduce_is_the_sequential_sum(splits):
    n = 8 * sms() * 1024 + 4 * 37                                # the grid-stride loop runs twice; not a multiple of 1024
    part = torch.randn(splits, n, device="cuda") * torch.exp2(torch.randint(-8, 9, (splits, 1), device="cuda").float())
    want = part[0].clone()
    for z in range(1, splits):
        want = want + part[z]
    assert_same_bits(ops.splitk_reduce(part), want, f"splitk_reduce, {splits} splits")
    for k in (0, 3, 10):
        alpha = torch.tensor([2.0 ** -k], device="cuda")
        assert_same_bits(ops.splitk_reduce(part, alpha=alpha), want * alpha, f"splitk_reduce, {splits} splits, alpha 2^-{k}")


# ------------------------------------------------------------------------------ re-layouts
PATCH_CASES = [(2, 3, 32, 48, 8, 4), (3, 1, 24, 16, 6, 8), (2, 4, 40, 24, 5, 12), (1, 3, 16, 16, 16, 16), (4, 3, 64, 32, 8, 8)]


@pytest.mark.parametrize("B,C,Hh,W,ph,pw", PATCH_CASES)
def test_patchify_unpatchify_are_torch_permutes(B, C, Hh, W, ph, pw):
    img = torch.randn(B, C, Hh, W, device="cuda")
    ref = img.view(B, C, Hh // ph, ph, W // pw, pw).permute(0, 2, 4, 1, 3, 5).reshape(B * (Hh // ph) * (W // pw), C * ph * pw)
    p = ops.patchify(img, (ph, pw), False)
    assert_same_bits(p, ref, "patchify vs reshape / permute")
    assert_same_bits(ops.patchify(img, (ph, pw), True), tf32_rn(ref), "patchify round_out vs tf32_rn")
    assert_same_bits(ops.unpatchify(p, None, B, C, Hh, W, (ph, pw)), img, "unpatchify(patchify(x))")
    bias = torch.randn(C, device="cuda")
    tok = torch.randn_like(p)
    want = tok.view(B, Hh // ph, W // pw, C, ph, pw).permute(0, 3, 1, 4, 2, 5).reshape(B, C, Hh, W) + bias.view(1, C, 1, 1)
    assert_same_bits(ops.unpatchify(tok, bias, B, C, Hh, W, (ph, pw)), want, "unpatchify with bias vs permute + bias")


@pytest.mark.parametrize("M,R,D", [(1000, 384, 64), (77, 1, 260), (5, 12, 4), ("two_passes+3", 1024, 8)])
def test_add_rows_mod_is_torch_indexing(M, R, D):
    if M == "two_passes+3":                                        # 8 SMs CTAs of 256 float4 per grid pass
        M = 2 * 8 * sms() * 256 * 4 // D + 3
    x, table = torch.randn(M, D, device="cuda"), torch.randn(R, D, device="cuda")
    assert_same_bits(ops.add_rows_mod(x, table), x + table[torch.arange(M, device="cuda") % R], f"add_rows_mod M {M} R {R}")


# ------------------------------------------------------------------------------ grad_scale
def expected_scale(m, t):
    if m == 0 or not math.isfinite(m):
        return 1.0, 1.0
    f, e = math.frexp(m)
    if f == 0.5:
        e -= 1                                                    # m = 2^e exactly
    sh = max(-100, min(100, t - e))
    return 2.0 ** sh, 2.0 ** -sh


def check_scale(g, t, what):
    m = g.abs().max().item()
    got = ops.grad_scale(g, t).tolist()
    want = expected_scale(m, t)
    assert got == list(want), f"{what}: grad_scale = {got}, want {list(want)} (max|g| {m!r} = {m.hex()}, target 2^{t})"
    if want[0] != 1.0 and abs(math.log2(want[0])) < 100:
        assert 2.0 ** (t - 1) < m * want[0] <= 2.0 ** t, what


@pytest.mark.parametrize("t", [-14, 6, 15])
@pytest.mark.parametrize("where", ["first", "last", "past_pass"])
def test_grad_scale_power_of_two_and_neighbours(where, t):
    n = 2 * absmax_pass() + 8
    pos = {"first": 0, "last": n - 1, "past_pass": absmax_pass() + 3}[where]
    for k in (-20, -1, 0, 3, 17):
        for top, name in ((2.0 ** k, "2^k"), (2.0 ** k * (1 + 2.0 ** -23), "just above 2^k"), (2.0 ** k * (1 - 2.0 ** -24), "just below 2^k")):
            g = (torch.rand(n, device="cuda") * 2 - 1) * (2.0 ** (k - 1))
            g[pos] = -top if k % 2 else top
            check_scale(g, t, f"max|g| {name}, k {k}, at {where}")


@pytest.mark.parametrize("t", [-14, 15])
def test_grad_scale_clamps_the_exponent(t):
    g = torch.zeros(4096, device="cuda")
    for v in (2.0 ** -140 * 1.5, 2.0 ** -149, 2.0 ** -126 * 0.75):   # subnormal max|g|
        g[100] = v
        check_scale(g, t, f"subnormal max {v!r}")
    for v in (2.0 ** 120, 3.0e38):
        g[100] = -v
        check_scale(g, t, f"huge max {v!r}")


@pytest.mark.parametrize("special", ["zero", "inf", "-inf", "nan", "-nan"])
@pytest.mark.parametrize("where", ["first", "last", "past_pass"])
def test_grad_scale_zero_inf_nan_give_one(where, special):
    n = 2 * absmax_pass() + 8
    pos = {"first": 0, "last": n - 1, "past_pass": absmax_pass() + 3}[where]
    g = torch.randn(n, device="cuda")
    if special == "zero":
        g.zero_()
    else:
        g[pos:pos + 1] = from_bits({"inf": 0x7F800000, "-inf": 0xFF800000, "nan": 0x7FC00000, "-nan": 0xFFFFFFFF}[special])
    assert ops.grad_scale(g).tolist() == [1.0, 1.0], f"{special} at {where}"
