"""The checkers of tests/exact_ref.py have teeth: fed mutated fp64 "kernel outputs" of a convolution, each mutation a kernel could
plausibly make is flagged, while the global metric of the older tests (max |out - ref| / max |ref| < 1.5e-2) lets the truncating
store and the one-ulp element through.  Also cross-checks the fp64 tap-decomposition references against torch's fp64 convolution,
and the fp32 BatchNorm restatements against fp64 autograd of batch_norm (+ residual, + ReLU), with their own mutations."""
import math

import numpy as np
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


# ---------------------------------------------------------------------------------------------------------------------
# PS update restatements (aggregate_update.cu sources and optimizer tail, cast_params, cyclic projection)
# ---------------------------------------------------------------------------------------------------------------------
U = 2.0 ** -24            # unit roundoff of fp32


def _np(seed):
    return np.random.default_rng(seed)


def _sgd_bound_step(e_p, e_m, p, m, d_in, *, lr, mu, c, wd, nesterov, first):
    """One step of the first-order error recurrence of ``sgd_tail_ref`` against exact arithmetic, element-wise in fp64.
    Each rounding contributes at most U times the magnitude it rounds, each fp32 coefficient (lr, mu, wd, c) U times its term:

        e_d = |wd| e_p + 2U (|wd p| + |d|)
        e_b = e_d (first step)  or  mu e_m + c e_d + 4U (mu |m| + |c d|)
        e_n = mu e_b + e_d + 2U (mu |b| + |d|)   (Nesterov; else e_n = e_b, and e_n = e_d without momentum)
        e_p' = e_p + lr e_n + 3U (|p| + lr |n|)
    Magnitudes are those of the fp64 trajectory; the test doubles the bound for the second-order terms."""
    d = d_in + wd * p
    e_d = abs(wd) * e_p + (2 * U * (np.abs(wd * p) + np.abs(d)) if wd else 0.0)
    if mu:
        if first:
            b, e_b = d, e_d
        else:
            b = mu * m + c * d
            e_b = mu * e_m + c * e_d + 4 * U * (mu * np.abs(m) + np.abs(c * d))
        n, e_n = (mu * b + d, mu * e_b + e_d + 2 * U * (mu * np.abs(b) + np.abs(d))) if nesterov else (b, e_b)
        m, e_m = b, e_b
    else:
        n, e_n = d, e_d
    return e_p + lr * e_n + 3 * U * (np.abs(p) + lr * np.abs(n)), e_m


@pytest.mark.parametrize("mu,damp,wd,nesterov", [(0.0, 0.0, 0.0, False), (0.9, 0.0, 5e-4, True), (0.9, 0.1, 5e-4, False),
                                                 (0.9, 0.5, 0.0, False)])
def test_sgd_restatement_tracks_fp64_torch_sgd(mu, damp, wd, nesterov):
    """200 steps of ``sgd_tail_ref`` in fp32 against torch.optim.SGD in fp64 on the same fp32 gradients: every element of
    params and momentum stays within twice the bound of ``_sgd_bound_step``."""
    rng = _np(1)
    n, lr = 4096, 0.05
    p32 = rng.standard_normal(n).astype(np.float32)
    m32 = np.zeros(n, np.float32)
    p64 = torch.tensor(p32.astype(np.float64), requires_grad=True)
    opt = torch.optim.SGD([p64], lr=lr, momentum=mu, dampening=damp, weight_decay=wd, nesterov=nesterov)
    e_p = e_m = np.zeros(n)
    c = float(X.one_minus_f32(damp))
    for t in range(200):
        g = (rng.standard_normal(n) * 0.1).astype(np.float32)
        pr = p64.detach().numpy().copy()
        mr = opt.state[p64]["momentum_buffer"].numpy().copy() if t and mu else np.zeros(n)
        e_p, e_m = _sgd_bound_step(e_p, e_m, pr, mr, g.astype(np.float64), lr=lr, mu=mu, c=c, wd=wd, nesterov=nesterov,
                                   first=t == 0)
        p32, m32 = X.sgd_tail_ref(g, p32, m32, lr=lr, momentum=mu, dampening=damp, weight_decay=wd, nesterov=nesterov,
                                  first=t == 0)
        p64.grad = torch.from_numpy(g.astype(np.float64))
        opt.step()
    err = np.abs(p32 - p64.detach().numpy())
    assert (err <= 2 * e_p).all(), f"params: worst err/bound {float((err / (2 * e_p)).max()):.3f}"
    if mu:
        err_m = np.abs(m32 - opt.state[p64]["momentum_buffer"].numpy())
        assert (err_m <= 2 * e_m + 1e-300).all(), f"momentum: worst err/bound {float((err_m / (2 * e_m)).max()):.3f}"


@pytest.mark.parametrize("amsgrad", [False, True])
def test_adam_restatement_tracks_fp64_torch_adam(amsgrad):
    """200 steps of ``adam_tail_ref`` in fp32 against torch.optim.Adam in fp64.  torch adds eps after dividing sqrt(v) by
    sqrt(1 - beta2^t); the kernel (like the reference's AdamModified) folds the corrections into the step size and adds eps to
    sqrt(v) itself, so eps = 1e-30 here makes the two formulas agree to far below fp32 resolution.  Per element and step, with
    e_d as for SGD, r = m / (sqrt(s) + eps) and a = the step size (all magnitudes from the fp64 trajectory):

        e_m = b1 e_m + c1 e_d + 4U (b1 |m| + c1 |d|)
        e_v = b2 e_v + c2 (2 |d| e_d + e_d^2) + 5U (b2 v + c2 d^2);   AMSGrad: e_s = max(e_s, e_v)
        e_sqrt = min(e_s / (2 sqrt(s)), sqrt(e_s)) + U sqrt(s);   e_r = e_m / sqrt(s) + |r| e_sqrt / sqrt(s) + U |r|
        e_p' = e_p + a e_r + 2U a |r| + 2U (|p| + a |r|)
    and every element of params, m, v (and vmax) stays within twice that bound."""
    rng = _np(2)
    n, lr, b1, b2, wd = 4096, 1e-3, 0.9, 0.999, 1e-4
    p32 = rng.standard_normal(n).astype(np.float32)
    m32, v32, vm32 = (np.zeros(n, np.float32) for _ in range(3))
    p64 = torch.tensor(p32.astype(np.float64), requires_grad=True)
    opt = torch.optim.Adam([p64], lr=lr, betas=(b1, b2), eps=1e-30, weight_decay=wd, amsgrad=amsgrad)
    e_p, e_m, e_v, e_s = (np.zeros(n) for _ in range(4))
    c1, c2 = float(X.one_minus_f32(b1)), float(X.one_minus_f32(b2))
    m = v = vm = np.zeros(n)
    for t in range(1, 201):
        g = (rng.standard_normal(n) * 0.1 * (1 + (t % 7))).astype(np.float32)
        p = p64.detach().numpy().copy()
        d = g.astype(np.float64) + wd * p
        e_d = wd * e_p + 2 * U * (np.abs(wd * p) + np.abs(d))
        e_m = b1 * e_m + c1 * e_d + 4 * U * (b1 * np.abs(m) + c1 * np.abs(d))
        e_v = b2 * e_v + c2 * (2 * np.abs(d) * e_d + e_d ** 2) + 5 * U * (b2 * v + c2 * d * d)
        m, v = b1 * m + (1 - b1) * d, b2 * v + (1 - b2) * d * d
        vm = np.maximum(vm, v)
        s = vm if amsgrad else v
        e_s = np.maximum(e_s, e_v) if amsgrad else e_v
        rs = np.sqrt(s)
        e_sqrt = np.minimum(e_s / (2 * rs), np.sqrt(e_s)) + U * rs
        r = m / rs
        e_r = e_m / rs + np.abs(r) * e_sqrt / rs + U * np.abs(r)
        a = lr * math.sqrt(1 - b2 ** t) / (1 - b1 ** t)
        e_p = e_p + a * e_r + 2 * U * a * np.abs(r) + 2 * U * (np.abs(p) + a * np.abs(r))
        step = X.adam_step_size_ref(lr, b1, b2, t)
        p32, m32, v32, vm32 = X.adam_tail_ref(g, p32, m32, v32, vm32, step_size=step, beta1=b1, beta2=b2, eps=1e-30,
                                              weight_decay=wd, amsgrad=amsgrad)
        p64.grad = torch.from_numpy(g.astype(np.float64))
        opt.step()
    st = opt.state[p64]
    for name, got, want, bound in (("params", p32, p64.detach().numpy(), e_p), ("exp_avg", m32, st["exp_avg"].numpy(), e_m),
                                   ("exp_avg_sq", v32, st["exp_avg_sq"].numpy(), e_v)) + (
            (("max_exp_avg_sq", vm32, st["max_exp_avg_sq"].numpy(), e_s),) if amsgrad else ()):
        err = np.abs(got.astype(np.float64) - want)
        assert (err <= 2 * bound).all(), f"{name}: worst err/bound {float((err / (2 * bound)).max()):.3f}"


def _ulps(got, want, scale=None) -> float:
    """max |got - want| in fp32 ulps of ``scale`` (default: of want)."""
    want = np.asarray(want, dtype=np.float64)
    ulp = X.ulp_f32(torch.from_numpy(want if scale is None else np.asarray(scale, np.float64))).numpy()
    return float((np.abs(np.asarray(got, np.float64) - want) / ulp).max())


@pytest.mark.parametrize("amsgrad", [False, True])
def test_restatements_match_library_optimizers_on_identical_aggregates(amsgrad):
    """One step of the restatements and of SGDModified / AdamModified (the library PS, fp32 tensors) from the same state and
    the same aggregate, at a fresh state (t = 1, v = 0) and at t = 2, 3, 10: params, momentum, exp_avg_sq and max_exp_avg_sq
    agree within 4 fp32 ulp of the magnitudes they are formed from (the library rounds b1 m and c1 d apart where the kernel
    fuses them, so a sum that cancels differs in more of its own ulps).  The library forms 1 - beta in fp64 and rounds it once, and takes the fp64 betas in the bias
    corrections; a kernel that forms them in fp32 misses by about 100 ulp in v at t = 1."""
    from draco_b200.optim import AdamModified, SGDModified
    rng = _np(3)
    n = 8192
    p0 = (rng.standard_normal(n) * 1e-4).astype(np.float32)          # small params: the step itself is visible to the ulp
    for t in (1, 2, 3, 10):
        g = (rng.standard_normal(n) * 0.1).astype(np.float32)
        m0 = (rng.standard_normal(n) * 0.01).astype(np.float32) if t > 1 else np.zeros(n, np.float32)
        v0 = (rng.random(n) * 1e-3).astype(np.float32) if t > 1 else np.zeros(n, np.float32)
        vm0 = (v0 * rng.choice([0.5, 2.0], n)).astype(np.float32)
        pt = torch.from_numpy(p0.copy())
        opt = AdamModified([pt], lr=1e-3, weight_decay=1e-4, amsgrad=amsgrad)
        opt.step([torch.zeros(n)])                                      # create the state, then overwrite it
        st = opt.state[pt]
        pt.copy_(torch.from_numpy(p0))
        st["step"], st["exp_avg"], st["exp_avg_sq"] = t - 1, torch.from_numpy(m0.copy()), torch.from_numpy(v0.copy())
        if amsgrad:
            st["max_exp_avg_sq"] = torch.from_numpy(vm0.copy())
        opt.step([torch.from_numpy(g)])
        p, m, v, vm = X.adam_tail_ref(g, p0, m0, v0, vm0, step_size=X.adam_step_size_ref(1e-3, 0.9, 0.999, t), beta1=0.9,
                                      beta2=0.999, eps=1e-8, weight_decay=1e-4, amsgrad=amsgrad)
        # ulps of the magnitudes each result is formed from (m and p may cancel): M = |b1 m| + |c1 d|, V = b2 v + c2 d^2,
        # P = |p| + a M / (sqrt(s) + eps)
        d = np.abs(g.astype(np.float64) + 1e-4 * p0)
        M = 0.9 * np.abs(m0) + 0.1 * d
        V = 0.999 * v0 + 1e-3 * d * d
        s_ = np.maximum(V, vm0) if amsgrad else V
        P = np.abs(p0) + float(X.adam_step_size_ref(1e-3, 0.9, 0.999, t)) * M / (np.sqrt(s_) + 1e-8)
        for name, got, want, mag in (("params", p, pt, P), ("exp_avg", m, st["exp_avg"], M),
                                     ("exp_avg_sq", v, st["exp_avg_sq"], V)) + (
                (("max_exp_avg_sq", vm, st["max_exp_avg_sq"], np.maximum(V, vm0)),) if amsgrad else ()):
            assert _ulps(got, want.numpy(), mag) <= 4, f"t={t} {name}: {_ulps(got, want.numpy(), mag)} ulp"
    for damp, nest in ((0.0, True), (0.1, False), (0.3, False)):
        g = (rng.standard_normal(n) * 0.1).astype(np.float32)
        pt = torch.from_numpy(p0.copy())
        opt = SGDModified([pt], lr=0.05, momentum=0.9, dampening=damp, weight_decay=5e-4, nesterov=nest)
        m0 = np.zeros(n, np.float32)
        for first in (True, False):
            p_prev = pt.numpy().copy()
            opt.step([torch.from_numpy(g)])
            p, m0 = X.sgd_tail_ref(g, p_prev, m0, lr=0.05, momentum=0.9, dampening=damp, weight_decay=5e-4, nesterov=nest,
                                   first=first)
            mom = opt.state[pt]["momentum_buffer"].numpy()
            Mg = np.abs(g) + 5e-4 * np.abs(p_prev) + 0.9 * np.abs(mom)              # the magnitudes m and p are formed from
            assert _ulps(m0, mom, Mg) <= 4 and _ulps(p, pt.numpy(), np.abs(p_prev) + 0.05 * 1.9 * Mg) <= 4, (damp, first)


def _old_close(got, want, atol) -> bool:
    """The older GPU tests' check: allclose with an absolute tolerance (NaN where both are NaN counts as equal)."""
    return bool(torch.allclose(torch.from_numpy(np.asarray(got, np.float64)), torch.from_numpy(np.asarray(want, np.float64)),
                               atol=atol, rtol=0, equal_nan=True))


def _differs(a, b) -> bool:
    return bool(X.mismatch(torch.from_numpy(np.asarray(a, np.float32)), torch.from_numpy(np.asarray(b, np.float32))))


def test_ps_update_exact_checks_flag_every_mutant():
    """Mutated restatements of the update kernel's sources, optimizer tail and cast, each flagged by the exact comparison.
    The older tests' tolerances (atol 1e-5 on params, 1e-6 on the aggregate, 5e-5 on the cyclic decode, torch.equal on the
    cast) accept the ones listed at the end on this data (params of 1e-4, steps of 1e-3): weight decay after momentum, the fp32
    1 - beta of the kernel before the fix, mode 0 dividing by K and an unfused mode 1.  The others move params by more than
    1e-5 here, though at other scales (smaller lr, larger params) the old tolerances would take them too."""
    rng = _np(4)
    n = 8192
    g = (rng.standard_normal(n) * 0.1).astype(np.float32)
    p0 = (rng.standard_normal(n) * 1e-4).astype(np.float32)
    m0 = (rng.standard_normal(n) * 0.01).astype(np.float32)
    v0 = (rng.random(n) * 1e-3).astype(np.float32)
    accepted = set()

    def note(name, got, want, atol):
        assert _differs(got, want), f"mutant '{name}' is not flagged"
        if atol is not None and _old_close(got, want, atol):
            accepted.add(name)

    # ---- SGD
    hp = dict(lr=0.05, momentum=0.9, weight_decay=5e-4)
    p_ok, _ = X.sgd_tail_ref(g, p0, m0, dampening=0.0, nesterov=True, first=False, **hp)
    p_mut, _ = X.sgd_tail_ref(g, p0, m0, dampening=0.0, nesterov=False, first=False, **hp)
    note("Nesterov dropped", p_mut, p_ok, 1e-5)
    p_ok, m_ok = X.sgd_tail_ref(g, p0, m0, dampening=0.1, nesterov=False, first=True, **hp)
    d = X._fma32(np.float32(5e-4), p0, g)
    b = X._mul32(X.one_minus_f32(0.1), d)                                           # dampening applied on the first step
    note("dampening on the first step", X._fma32(-np.float32(0.05), b, p0), p_ok, 1e-5)
    p_ok, m_ok = X.sgd_tail_ref(g, p0, m0, dampening=0.0, nesterov=False, first=False, **hp)
    b = X._fma32(np.float32(0.9), m0, g)                                            # weight decay after momentum
    note("weight decay after momentum", X._fma32(-np.float32(0.05), X._fma32(np.float32(5e-4), p0, b), p0), p_ok, 1e-5)
    # ---- Adam / AMSGrad
    ad = dict(beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=1e-4)
    vm0 = (v0 * rng.choice([0.5, 2.0], n)).astype(np.float32)
    step3 = X.adam_step_size_ref(1e-3, 0.9, 0.999, 3)
    ok = X.adam_tail_ref(g, p0, m0, v0, vm0, step_size=step3, amsgrad=True, **ad)
    dd = X._fma32(np.float32(1e-4), p0, g)
    mm = X._fma32(np.float32(0.9), m0, X._mul32(X.one_minus_f32(0.9), dd))
    vmax_early = np.fmax(vm0, v0)                                                   # the max taken before the v update
    u = X._div32(mm, X._add32(X._sqrt32(vmax_early), np.float32(1e-8)))
    note("AMSGrad max before the v update", X._fma32(-step3, u, p0), ok[0], 1e-5)
    vv = ok[2]
    u = X._div32(ok[1], X._sqrt32(X._add32(vv, np.float32(1e-8))))                  # eps inside the sqrt
    ok_adam = X.adam_tail_ref(g, p0, m0, v0, vm0, step_size=step3, amsgrad=False, **ad)
    note("eps inside the sqrt", X._fma32(-step3, u, p0), ok_adam[0], 1e-5)
    note("bias correction at t - 1", X.adam_tail_ref(g, p0, m0, v0, vm0, step_size=X.adam_step_size_ref(1e-3, 0.9, 0.999, 4),
                                                     amsgrad=False, **ad)[0], ok_adam[0], 1e-5)
    # fp32 1 - beta and fp32 betas in the bias corrections (the kernel before the fix), at a fresh state
    z = np.zeros(n, np.float32)
    fresh = X.adam_tail_ref(g, p0, z, z, z, step_size=X.adam_step_size_ref(1e-3, 0.9, 0.999, 1), amsgrad=False, **ad)
    b1f, b2f = np.float32(0.9), np.float32(0.999)
    step_f32b = np.float32(float(np.float32(1e-3)) * math.sqrt(1 - float(b2f)) / (1 - float(b1f)))
    mut = X.adam_tail_ref(g, p0, z, z, z, step_size=step_f32b, amsgrad=False, c1=np.float32(1) - b1f, c2=np.float32(1) - b2f, **ad)
    assert _differs(mut[2], fresh[2]) and _differs(mut[0], fresh[0])
    note("fp32 1 - beta", mut[0], fresh[0], 1e-5)
    # ---- sources
    for Kr in (3, 7):
        rows = (rng.standard_normal((Kr, n)) * 0.1).astype(np.float32)
        sc = np.float32(1.0 / Kr)
        ok = X.update_source_ref(0, rows, sc)
        acc = rows[0]
        for k in range(1, Kr):
            acc = X._add32(acc, rows[k])
        note("mode 0 dividing by K", X._div32(acc, np.float32(Kr)), ok, 1e-6)
    nr = 7
    cre, cim = (rng.standard_normal((nr, n)).astype(np.float32) for _ in range(2))
    v = (rng.standard_normal(nr) + 1j * rng.standard_normal(nr)).astype(np.complex64)
    v[2] = 0
    ok = X.update_source_ref(1, (cre, cim), np.float32(1 / nr), recomb=v)
    acc = np.zeros(n, np.float32)
    for k in range(nr):
        if v[k] != 0:
            acc = X._add32(acc, X._add32(X._mul32(v[k].real, cre[k]), -X._mul32(v[k].imag, cim[k])))
    note("mode 1 unfused", X._mul32(acc, np.float32(1 / nr)), ok, 5e-5)
    # ---- cast: truncation in place of round-to-nearest-even
    x = (rng.standard_normal(n) * 3).astype(np.float32)
    trunc = (x.view(np.uint32) >> 16).astype(np.uint16)
    assert (trunc != X.cast_bf16_ref(x)).any()
    rne = torch.from_numpy(X.cast_bf16_ref(x).view(np.int16)).view(torch.bfloat16)
    if torch.equal(torch.from_numpy(trunc.view(np.int16)).view(torch.bfloat16), rne):
        accepted.add("truncating bf16 cast")
    print("mutants the older tolerances accept:", sorted(accepted))
    assert accepted == {"weight decay after momentum", "fp32 1 - beta", "mode 0 dividing by K", "mode 1 unfused"}, accepted


def test_update_source_and_cast_restatements_on_edges():
    """The sources on +-0, subnormals and NaN / Inf rows, and the cast on ties, subnormals, overflow and zeros, against
    independent formulations: torch's fp32 -> bf16 conversion and sums accumulated one fp32 add at a time."""
    x = np.array([1.0, 1 + 2 ** -8, 1 + 3 * 2 ** -8, -(1 + 2 ** -8), 3.3961e38, 3.4e38, -3.4e38, 1e-40, -1e-40, 2 ** -133,
                  3 * 2 ** -134, -0.0, 0.0, np.inf, -np.inf, np.nan], np.float32)
    r = X.cast_bf16_ref(x)
    t = torch.from_numpy(x).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    fin = ~np.isnan(x)
    assert (r[fin] == t[fin]).all() and np.isnan(torch.from_numpy(r.view(np.int16)).view(torch.bfloat16).float().numpy()[~fin]).all()
    rng = _np(5)
    x = torch.from_numpy((rng.standard_normal(100000) * 100).astype(np.float32))
    assert (X.cast_bf16_ref(x.numpy()) == x.to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)).all()
    rows = np.array([[-0.0, -0.0, 1e-45, np.inf, np.nan, 3e38], [-0.0, 0.0, 1e-45, -np.inf, 1.0, 3e38]], np.float32)
    g = X.update_source_ref(0, rows, 0.5)
    assert np.signbit(g[0]) == False and g[1] == 0 and g[2] == np.float32(1e-45)        # -0 + -0 from +0 is +0; 2 ulp * 0.5
    assert np.isnan(g[3]) and np.isnan(g[4]) and g[5] == np.inf                         # Inf - Inf, NaN, overflow
    w = X.update_source_ref(2, rows, 1.0, weights=np.array([0.5, 0.5], np.float32))
    # fma(0.5, 2^-149, 0) is a tie between 0 and 2^-149 and rounds to the even 0, twice; fma(0.5, 3e38, 1.5e38) does not overflow
    assert w[2] == 0 and w[5] == np.float32(3e38)


def test_cyclic_project_reference_is_the_fp64_projection():
    """``cyclic_project_ref`` sums the same products as an fp64 dot product, only in the kernels' order: within 1e-12."""
    rng = _np(6)
    ntiles, n = 70, 5
    tile_tensor = np.repeat(np.arange(4), [3, 1, 33, 33])
    numel = [2500, 20, 33 * 1024 - 7, 32 * 1024 + 1]
    valid = np.concatenate([np.clip(nl - 1024 * np.arange(c), 0, 1024) for nl, c in zip(numel, [3, 1, 33, 33])])
    mask = (np.arange(1024)[None, :] < valid[:, None]).reshape(-1)
    Rr, Ri = ((rng.standard_normal((n, ntiles * 1024)) * mask).astype(np.float32) for _ in range(2))
    f = ((rng.standard_normal(ntiles * 1024) + 1) * mask).astype(np.float32)
    Er, Ei = X.cyclic_project_ref(Rr, Ri, f, tile_tensor, valid)
    for t in range(4):
        sl = np.repeat(tile_tensor == t, 1024)
        for E, R in ((Er, Rr), (Ei, Ri)):
            ref = R[:, sl].astype(np.float64) @ f[sl].astype(np.float64)
            assert np.abs(E[t] - ref).max() <= 1e-12 * (np.abs(R[:, sl].astype(np.float64)) @ np.abs(f[sl].astype(np.float64))).max()
