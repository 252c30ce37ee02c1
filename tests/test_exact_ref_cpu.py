"""The checkers of tests/exact_ref.py have teeth: fed mutated fp64 "kernel outputs" of a convolution, each mutation a kernel could
plausibly make is flagged, while the global metric of the older tests (max |out - ref| / max |ref| < 1.5e-2) lets the truncating
store and the one-ulp element through.  Also cross-checks the fp64 tap-decomposition references against torch's fp64 convolution."""
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
