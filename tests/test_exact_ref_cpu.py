"""The checkers of tests/exact_ref.py have teeth: fed mutated fp64 "kernel outputs" of a convolution, each mutation a kernel could
plausibly make is flagged, while the global metric of the older tests (max |out - ref| / max |ref| < 1.5e-2) lets the truncating
store and the one-ulp element through.  Also cross-checks the fp64 tap-decomposition references against torch's fp64 convolution,
and the fp32 BatchNorm restatements against fp64 autograd of batch_norm (+ residual, + ReLU), with their own mutations."""
import pytest
import torch
import torch.nn.functional as F

import exact_ref as X

OLD_TOL = 1.5e-2


def _gen(seed):
    g = torch.Generator()
    g.manual_seed(seed)
    return g


@pytest.mark.parametrize("n,cin,cout,h,w,ks,stride", [(2, 5, 7, 6, 10, 3, 1), (3, 4, 6, 8, 6, 3, 2), (2, 3, 5, 6, 4, 1, 2),
                                                      (1, 6, 4, 7, 5, 3, 1)])
def test_fp64_references_match_torch(n, cin, cout, h, w, ks, stride):
    g = _gen(n + cin + h)
    x = torch.randn(n, cin, h, w, generator=g, dtype=torch.float64)
    wt = torch.randn(cout, cin, ks, ks, generator=g, dtype=torch.float64)
    b = torch.randn(cout, generator=g, dtype=torch.float64)
    oh, ow = h // stride, w // stride
    xs = x[:, :, :oh * stride, :ow * stride] if (h % stride or w % stride) else x
    y = X.conv_ref(xs, wt, stride, b)
    assert torch.allclose(y, F.conv2d(xs, wt, b, stride=stride, padding=ks // 2), rtol=1e-12, atol=1e-12)
    dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
    hw = (oh * stride, ow * stride)
    dx = X.dgrad_ref(dy, wt, hw, stride)
    assert torch.allclose(dx, torch.nn.grad.conv2d_input((n, cin) + hw, wt, dy, stride=stride, padding=ks // 2), rtol=1e-12, atol=1e-12)
    dw = X.wgrad_ref(dy, xs, ks, stride)
    assert torch.allclose(dw, torch.nn.grad.conv2d_weight(xs, wt.shape, dy, stride=stride, padding=ks // 2), rtol=1e-12, atol=1e-12)


def test_bf16_rounding_helpers():
    v = torch.tensor([1.0, 257.0, 258.0, 259.0, 1026.0, 1030.0, -1030.0, 1.0 + 2 ** -8, 1.0 + 3 * 2 ** -9, 0.0, 3.0e38 / 2 ** 100],
                     dtype=torch.float64)
    rn = X.bf16_rn(v)
    # ties go to the even significand: 257 -> 256, 259 -> 260, 1030 -> 1032 (1024 + 3 * 2 ties to 1024 + 4 * 2)
    assert rn.double().tolist()[:9] == [1.0, 256.0, 258.0, 260.0, 1024.0, 1032.0, -1032.0, 1.0, 1.0 + 2 ** -7]
    # the helper rounds fp64 once: agrees with torch's (fp32-mediated) conversion wherever the fp64 value is an fp32
    r = torch.randn(10000, dtype=torch.float64).float().double() * 100
    assert torch.equal(X.bf16_rn(r), r.to(torch.bfloat16))
    assert torch.equal(X.bf16_rz(v).double()[:4], torch.tensor([1.0, 256.0, 258.0, 258.0], dtype=torch.float64))
    assert X.ulp_bf16(torch.tensor([1.0, 1.5, 1024.0])).tolist() == [2 ** -7, 2 ** -7, 8.0]


def test_integer_operands_are_exact_in_fp32():
    """The premise of the exact tests: at K = 9 * 512 an fp32 convolution of {-1, 0, 1} operands equals the fp64 one."""
    g = _gen(3)
    K = 9 * 512
    x = X.int_operand((4, 512, 4, 4), K, g)
    w = X.int_operand((512, 512, 3, 3), K, g)
    y32 = X.conv_ref(x.float(), w.float(), 1).float()          # fp64 accumulation of the same integers
    y32_direct = F.conv2d(x, w, padding=1)                       # fp32 accumulation, library order
    assert torch.equal(y32_direct.double(), X.conv_ref(x, w, 1))
    assert torch.equal(y32.double(), X.conv_ref(x, w, 1))
    assert 0 < float(y32.abs().max()) < 2 ** 11
    assert X.density_for(K) == pytest.approx((2 ** 11 / K) ** 0.5)


# ------------------------------------------------------------------------------------------------------------------------------
# mutations of a convolution output: n = 13 images 4 x 4 (208 pixel rows: the second 128-row tile is partial), 512 -> 512, 3x3
# ------------------------------------------------------------------------------------------------------------------------------
N, C, HW = 13, 512, 4


@pytest.fixture(scope="module")
def int_case():
    g = _gen(11)
    K = 9 * C
    x = X.int_operand((N, C, HW, HW), K, g)
    w = X.int_operand((C, C, 3, 3), K, g)
    bias = (1000 + torch.arange(C) % 37).double() * (1 - 2 * (torch.arange(C) % 2))     # +-1000 + k: outputs need rounding
    ref = X.conv_ref(x, w, 1, bias)
    return x, w, bias, ref, X.bf16_rn(ref)


@pytest.fixture(scope="module")
def real_case():
    g = _gen(12)
    x = torch.randn(N, C, HW, HW, generator=g).to(torch.bfloat16).double()                 # the data scaling of the older tests
    w = (torch.randn(C, C, 3, 3, generator=g) * 0.05).to(torch.bfloat16).double()
    ref = X.conv_ref(x, w, 1)
    absref = X.conv_ref(x.abs(), w.abs(), 1)
    return x, w, ref, absref, X.bf16_rn(ref)


def _mutations(x, w, ref, good, bias=None):
    """name -> mutated bf16 output (the same mutations for both cases)."""
    out = {}
    out["truncating store"] = X.bf16_rz(ref)
    one = good.clone()
    i = (0, 5, 1, 2)
    one[i] = X.bf16_rn(ref[i].reshape(1) + X.ulp_bf16(ref[i].reshape(1)) * (1.5 if ref[i] >= good[i].double() else -1.5))[0]
    out["one element off by one ulp"] = one
    rows = good.permute(0, 2, 3, 1).reshape(-1, C).clone()                  # NHWC pixel rows
    last = rows.shape[0] - 1                                                # row 207: last row of the partial tile 1
    rows[last] = rows[last - 1]
    out["last partial-tile row replaced by the row above"] = rows.reshape(N, HW, HW, C).permute(0, 3, 1, 2)
    w_drop = w.clone()
    w_drop[:, 17, 0, 2] = 0                                                 # input channel 17 of tap (0, 2) dropped
    out["one input channel of one tap dropped"] = X.bf16_rn(X.conv_ref(x, w_drop, 1, bias))
    return out


def _swapped_hw(x, w, bias):
    """A kernel that swaps H and W in its box / tile bookkeeping on a non-square input: it reads x [N, H, W, C] as if it were
    [N, W, H, C] and writes its result the same way."""
    n, c, h, wd = x.shape
    xs = x.permute(0, 2, 3, 1).reshape(n, wd, h, c).permute(0, 3, 1, 2)
    ys = X.conv_ref(xs, w, 1, bias)
    return X.bf16_rn(ys.permute(0, 2, 3, 1).reshape(n, h, wd, -1).permute(0, 3, 1, 2))


def test_exact_check_flags_every_mutation_the_old_metric_misses(int_case):
    x, w, bias, ref, good = int_case
    assert X.mismatch(good, X.bf16_rn(ref)) == ""
    muts = _mutations(x, w, ref, good, bias)
    for name, out in muts.items():
        assert X.mismatch(out, good), name
    # the global metric of the older tests cannot see the two rounding-level mutations
    assert X.rel_err(muts["truncating store"], ref) < OLD_TOL
    assert X.rel_err(muts["one element off by one ulp"], ref) < OLD_TOL
    # non-square input: H / W swapped
    g = _gen(5)
    xr = X.int_operand((3, 64, 4, 8), 9 * 64, g)
    wr = X.int_operand((64, 64, 3, 3), 9 * 64, g)
    ok = X.bf16_rn(X.conv_ref(xr, wr, 1))
    msg = X.mismatch(_swapped_hw(xr, wr, None), ok)
    assert msg and "pixel row" in msg and "tile" in msg


def test_component_bound_accepts_correct_and_flags_local_errors(real_case):
    x, w, ref, absref, good = real_case
    K = 9 * C
    assert X.bound_violation(good, ref, absref, K) == ""
    muts = _mutations(x, w, ref, good)
    # localized errors of a real-valued output are outside the per-element bound ...
    for name in ("last partial-tile row replaced by the row above", "one input channel of one tap dropped"):
        msg = X.bound_violation(muts[name], ref, absref, K)
        assert msg, name
    assert "tile 1" in X.bound_violation(muts["last partial-tile row replaced by the row above"], ref, absref, K)
    # ... while the rounding-level ones are only visible to the exact integer-operand check (see the test above)
    assert X.rel_err(muts["truncating store"], ref) < OLD_TOL
    g = _gen(6)
    xr = torch.randn(3, 64, 4, 8, generator=g).to(torch.bfloat16).double()
    wr = (torch.randn(64, 64, 3, 3, generator=g) * 0.05).to(torch.bfloat16).double()
    assert X.bound_violation(_swapped_hw(xr, wr, None), X.conv_ref(xr, wr, 1), X.conv_ref(xr.abs(), wr.abs(), 1), 9 * 64)


def test_batchnorm_statistics_reference_sees_one_masked_row():
    """With integer outputs the per-channel sums are exact: one mis-masked pixel row of a partial tile moves the mean, and the
    comparison is exact (the older tests' global metric normalised by the largest mean does not see it)."""
    g = _gen(8)
    y = torch.randint(-6, 7, (13, 64, 4, 4), generator=g).to(torch.bfloat16)
    m, var, invstd, rm, rv = X.bn_stats_ref(y, 1e-5, 0.1, torch.zeros(64), torch.ones(64))
    yb = y.clone()
    yb[12, :, 3, 3] = 0                                                   # last pixel row not counted
    mb, *_ = X.bn_stats_ref(yb, 1e-5, 0.1)
    assert not torch.equal(m, mb)
    # the fp32 emulation agrees with an fp64 computation to fp32 accuracy (m = S * fl(1/M) rounds twice: up to 1.5 ulp)
    yd = y.double()
    assert X.ulps_f32(m, yd.mean((0, 2, 3))) <= 1.5
    v64 = yd.var((0, 2, 3), unbiased=False)
    assert float(((var - v64).abs() / v64).max()) < 1e-5
    assert X.ulps_f32(rm, 0.1 * yd.mean((0, 2, 3))) <= 2


# ------------------------------------------------------------------------------------------------------------------------------
# BatchNorm apply and backward references (exact_ref.bn_*_ref)
# ------------------------------------------------------------------------------------------------------------------------------
U32 = 2.0 ** -24                                                          # unit roundoff of fp32


def _bn_real(M, c, seed, with_res):
    """bf16 activations [M, C] with one channel at a large mean / std ratio, fp32 parameters, the fp64 batch statistics and
    their fp32 roundings (what a convolution epilogue hands over)."""
    g = _gen(seed)
    off = torch.randn(c, generator=g, dtype=torch.float64) * 0.5
    off[1] = 60.0
    x = (torch.randn(M, c, generator=g, dtype=torch.float64) * 1.7 + off).to(torch.bfloat16)
    res = torch.randn(M, c, generator=g, dtype=torch.float64).to(torch.bfloat16) if with_res else None
    dy = torch.randn(M, c, generator=g, dtype=torch.float64).to(torch.bfloat16)
    gamma = (torch.rand(c, generator=g, dtype=torch.float64) + 0.5).float()
    beta = (torch.rand(c, generator=g, dtype=torch.float64) - 0.5).float()
    xd = x.double()
    mean64 = xd.mean(0)
    istd64 = 1.0 / (xd.var(0, unbiased=False) + 1e-5).sqrt()
    return x, res, dy, gamma, beta, mean64, istd64


@pytest.mark.parametrize("M,c", [(63, 5), (50, 7), (9, 3), (231, 16)])
@pytest.mark.parametrize("with_res", [False, True])
def test_bn_references_are_batchnorm_and_its_gradient(M, c, with_res):
    """bn_apply_ref and bn_bwd_apply_ref (fed with bn_bwd_sums_ref) against fp64 autograd of relu(batch_norm(x) + res).

    Per element, with u = 2^-24, gs = gamma * invstd, xhat = (x - mean) * invstd, m1 = mean(dz), m2 = mean(dz * xhat) (all
    exact fp64) and the fp32 statistics mean(1 + d), invstd(1 + d'), |d|, |d'| <= u:

      |y - y64|   <= ulp_bf16(y) / 2 + 8u (|gs| (|x| + |mean|) + |beta| + |res| + |y64|)
      |dx - dx64| <= ulp_bf16(dx) / 2 + 8u (|gs| (|dz| + |m1| + |xhat| (|m2| + mean|dz xhat| + |mean| invstd mean|dz|))
                                            + |gs m2 invstd| (|x| + |mean|))

    Half a bf16 ulp is the final rounding; every fp32 operation and the rounded statistics contribute O(u) relative to the
    magnitudes they touch (at most 6 roundings per term, 8 leaves slack).  The last term is the cancellation in cB x + cC
    when |mean| / std is large (channel 1 sits at mean / std ~ 35); the mean|dz xhat| and mean|dz| terms carry xhat's and the
    mean's fp32 roundings into m2.  Gradients are compared where both ReLU masks agree."""
    x, res, dy, gamma, beta, mean64, istd64 = _bn_real(M, c, M + c + with_res, with_res)
    mean32, istd32 = mean64.float(), istd64.float()
    xd = x.double().requires_grad_(True)
    rd = res.double().requires_grad_(True) if with_res else None
    gd, bd = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    y64 = F.batch_norm(xd, None, None, gd, bd, True, 0.1, 1e-5)
    pre = (y64 + rd) if with_res else y64
    y64 = F.relu(pre)
    y64.backward(dy.double())

    y, keep = X.bn_apply_ref(x, res, gamma, beta, mean32, istd32, True)
    gs = gamma.double() * istd64
    r_abs = res.double().abs() if with_res else 0.0
    bound_y = X.ulp_bf16(y) / 2 + 8 * U32 * (gs.abs() * (x.double().abs() + mean64.abs()) + beta.double().abs() + r_abs
                                            + pre.detach().abs())
    assert bool(((y.double() - y64.detach()).abs() <= bound_y).all())

    agree = keep == (y64.detach() > 0)
    assert float(agree.double().mean()) >= 0.99
    dz = torch.where(keep, dy, torch.zeros_like(dy))
    dbeta, dgamma, sums = X.bn_bwd_sums_ref(dz, x, mean32, istd32)
    dx, dres = X.bn_bwd_apply_ref(dy, keep, x, X.bn_bwd_coeffs_ref(gamma, istd32, mean32, sums))
    assert torch.equal(dres, dz)
    if with_res:
        X.assert_equal(dres.float()[agree], rd.grad.float()[agree], "dres")
    dzd = dz.double()
    xhat = (x.double() - mean64) * istd64
    m1, m2 = dzd.mean(0), (dzd * xhat).mean(0)
    a_dzx, a_dz = (dzd * xhat).abs().mean(0), dzd.abs().mean(0)
    bound_dx = X.ulp_bf16(dx) / 2 + 8 * U32 * (gs.abs() * (dzd.abs() + m1.abs() + xhat.abs() * (m2.abs() + a_dzx + mean64.abs() * istd64 * a_dz))
                                              + (gs * m2 * istd64).abs() * (x.double().abs() + mean64.abs()))
    err = (dx.double() - xd.grad).abs()
    assert bool((err <= bound_dx)[agree].all()), float((err / bound_dx)[agree].max())
    # dbeta = sum dz exactly; dgamma within the fp32 roundings of xhat and of the statistics
    assert torch.allclose(dbeta, bd.grad, rtol=1e-12, atol=1e-12)
    assert bool(((dgamma - gd.grad).abs() <= 8 * U32 * M * (a_dzx + mean64.abs() * istd64 * a_dz)).all())
    # sums are the fp32 means the coefficients are formed from
    assert X.ulps_f32(sums[:c], dbeta / M) <= 1.5 and X.ulps_f32(sums[c:], dgamma / M) <= 1.5


def _pack_bits(keep, reverse=False):
    """ReLU bits as bn_apply_kernel stores them: bit i of byte (row, cv) is channel 8 cv + i (bit 7 - i when ``reverse``)."""
    k = keep.reshape(keep.shape[0], -1, 8).long()
    sh = torch.arange(8)
    return (k << (7 - sh if reverse else sh)).sum(-1).to(torch.uint8).flatten()


def _old_accepts(out, ref, tol):
    """The older tests' global metric: max |out - ref| <= tol * max(1, max |ref|) (a NaN fails it)."""
    return float((out.double() - ref.double()).abs().max()) <= tol * max(1.0, float(ref.double().abs().max()))


def test_bn_exact_checks_flag_every_mutation_the_old_metric_misses():
    """Mutated restatements of the BatchNorm kernels, each flagged by the exact comparison.  Reduce-level mutations on integer
    data (x in [-8, 8], integer means, invstd = 1/4: the sums are exact), rounding-level ones on real data with NaN / Inf.
    The older tests' tolerances (2e-2 on y, 3e-2 on dx and dgamma, 99.5 % of mask bits) accept the listed ones."""
    g = _gen(21)
    M, c = 16384 + 5, 64
    x = torch.randint(-8, 9, (M, c), generator=g).to(torch.bfloat16)
    mean = torch.randint(-3, 4, (c,), generator=g).float()
    istd = torch.full((c,), 0.25)
    # gradients correlated with xhat, as a trained layer's are: dgamma ~ M, dbeta small
    noise = torch.randint(-1, 2, (M, c), generator=g)
    dy = torch.where(torch.rand(M, c, generator=g) < 0.7, torch.sign(x.float() - mean), noise.float()).to(torch.bfloat16)
    gamma = (torch.rand(c, generator=g) + 0.5)
    beta = (torch.rand(c, generator=g) - 0.5)
    y, keep = X.bn_apply_ref(x, None, gamma, beta, mean, istd, True)
    dz = torch.where(keep, dy, torch.zeros_like(dy))
    dbeta, dgamma, sums = X.bn_bwd_sums_ref(dz, x, mean, istd)
    co = X.bn_bwd_coeffs_ref(gamma, istd, mean, sums)
    dx, _ = X.bn_bwd_apply_ref(dy, keep, x, co)
    accepted = set()

    # one row dropped from the reduction (a remainder-loop bug): last row with a nonzero dz
    dz_drop = dz.clone()
    dz_drop[-1] = 0
    assert bool((dz[-1] != 0).any())
    _, dgamma_drop, sums_drop = X.bn_bwd_sums_ref(dz_drop, x, mean, istd)
    assert X.mismatch(dgamma_drop.float(), dgamma.float()) and X.mismatch(sums_drop, sums)
    if _old_accepts(dgamma_drop, dgamma, 3e-2):
        accepted.add("one dropped row in the sums")
    # 1 / (M - 1) in the sums
    inv = torch.tensor(1.0 / (M - 1), dtype=torch.float32).double()
    sums_m1 = torch.cat([dbeta * inv, dgamma * inv]).float()
    assert X.mismatch(sums_m1, sums)
    dx_m1, _ = X.bn_bwd_apply_ref(dy, keep, x, X.bn_bwd_coeffs_ref(gamma, istd, mean, sums_m1))
    assert X.mismatch(dx_m1, dx)
    if _old_accepts(dx_m1, dx, 3e-2):
        accepted.add("1/(M-1)")

    # real-valued data for the rounding-level mutations
    xr, res, dyr, gr, br, mean64, istd64 = _bn_real(M, c, 22, True)
    xr = xr.clone()
    xr.view(-1)[3::997] = float("nan")
    xr.view(-1)[5::1009] = float("inf")
    meanr, istdr = mean64.float(), istd64.float()
    yr, keepr = X.bn_apply_ref(xr, res, gr, br, meanr, istdr, True)
    assert not bool(yr.isnan().any())
    dzr = torch.where(keepr, dyr, torch.zeros_like(dyr)).float()
    sums_r = torch.cat([dzr.double().mean(0), dzr.double().mean(0) * 0.37 - 0.01]).float()    # any fp32 sums will do
    cA, cB, cC = X.bn_bwd_coeffs_ref(gr, istdr, meanr, sums_r)
    xrf = xr.float()
    dxr, _ = X.bn_bwd_apply_ref(dyr, keepr, xr, (cA, cB, cC))
    finite = torch.isfinite(dxr.float())
    # truncating bf16 store
    exact_pre = torch.from_numpy(X._fma32(cA.numpy(), dzr.numpy(), X._fma32(cB.numpy(), xrf.numpy(), cC.numpy())))
    dx_rz = X.bf16_rz(exact_pre.double())
    assert X.mismatch(dx_rz[finite], dxr[finite])
    if _old_accepts(dx_rz[finite], dxr[finite], 3e-2):
        accepted.add("truncating bf16 stores")
    # cB x + cC rounded before the outer fma
    unfused = (cB.double() * xrf.double()).float().double() + cC.double()
    dx_unf = X._bf16(X._fma32(cA.numpy(), dzr.numpy(), unfused.float().numpy()))
    assert X.mismatch(dx_unf, dxr)
    if _old_accepts(dx_unf[finite], dxr[finite], 3e-2):
        accepted.add("unfused cB*x + cC")
    # reversed bit order in the mask
    assert torch.equal(X.unpack_relu_bits(_pack_bits(keepr), (M, c)), keepr)
    rev = X.unpack_relu_bits(_pack_bits(keepr, reverse=True), (M, c))
    assert X.mismatch(rev, keepr)
    if float((rev == keepr).double().mean()) >= 0.995:
        accepted.add("reversed mask bits")
    # the pair's shortcut term formed with the main layer's mean
    xs = (torch.randn(M, c, generator=g) * 0.8 - 0.4).to(torch.bfloat16)
    gs_, bs_, ms_, is_ = torch.rand(c, generator=g) + 0.5, torch.rand(c, generator=g) - 0.5, xs.float().mean(0), torch.full((c,), 1.25)
    yp, _ = X.bn_apply_ref(xr, None, gr, br, meanr, istdr, True, pair=(xs, gs_, bs_, ms_, is_))
    yp_bad, _ = X.bn_apply_ref(xr, None, gr, br, meanr, istdr, True, pair=(xs, gs_, bs_, meanr, is_))
    assert X.mismatch(yp_bad, yp)
    if _old_accepts(yp_bad, yp, 2e-2):
        accepted.add("pair shortcut with the main mean")
    # a NaN-propagating ReLU in place of fmaxf
    y_lin, _ = X.bn_apply_ref(xr, res, gr, br, meanr, istdr, False)
    y_nan = torch.where(y_lin.isnan(), y_lin, y_lin.clamp_min(0))
    assert X.mismatch(y_nan, yr)
    if _old_accepts(y_nan, yr, 2e-2):
        accepted.add("NaN-propagating ReLU")
    assert accepted == {"one dropped row in the sums", "1/(M-1)", "truncating bf16 stores", "unfused cB*x + cC"}, accepted
