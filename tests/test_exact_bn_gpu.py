"""Exact tests of the BatchNorm apply and backward kernels (csrc/cuda/bn_fused.cu) through their C ABI and FusedBatchNorm2d.

The apply kernels are per-element functions of per-channel fp32 coefficients: on real data (with +-0, values that round to
bf16 zero, NaN and +-Inf) every output must equal the fp32 restatement in tests/exact_ref.py bit for bit (values compared, so
+0 == -0 and NaN == NaN).  The reductions are exact on integer data: dy in {-1, 0, 1}, x in [-8, 8], integer means and
invstd = 1/4 make every xhat a multiple of 1/4 and every partial sum an fp32 value, so dgamma, dbeta and both sums rows must
equal the fp64 sums in any order, for every grid plan.  Each reduction runs with num_sms in {1, 3, 7, the device's count,
1000}: the ticket reduction needs no co-residency, so every grid is valid, and the plans cover single-CTA and SM-capped
grids, partial last CTAs, rows_per_cta / row-group remainders and both grid_fold branches (C <= 1024 and C >= 2048).
"""
import zlib

import pytest
import torch

import exact_ref as X

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
THREADS = 512                                        # BN_THREADS: C / 8 lanes per row, 512 / (C / 8) row groups per CTA
CS = [8 << k for k in range(10)]                     # every supported C: 8 .. 4096
FLAGSHIP = [(131072, 64), (32768, 128), (8192, 256), (2048, 512)]     # ResNet-18 on 32 x 32 inputs, batch 128


def _rgroups(C):
    return THREADS // (C // 8)


def _ms(C):
    """M = 1; a few row groups plus a remainder (one CTA); and ~2^19 elements with M not a multiple of the row groups (C < 4096),
    which leaves the last CTA of the reduce grid partial at some num_sms."""
    rg = _rgroups(C)
    return [1, 3 * rg + 5, (1 << 19) // C + (rg + 1) // 2]


SHAPES = [(M, C) for C in CS for M in _ms(C)] + FLAGSHIP


def _sms_list():
    return [1, 3, 7, torch.cuda.get_device_properties(DEV).multi_processor_count, 1000]


def _plan(M, C, num_sms, reduce):
    """plan_rows of bn_fused.cu: (rows per CTA, grid)."""
    rg = _rgroups(C)
    target = max(1, min(-(-(M * C * 2) // 32768), num_sms if reduce else 4 * num_sms))
    rows = max(rg, -(-(-(-M // target)) // rg) * rg)
    return rows, -(-M // rows)


def test_plans_cover_partial_ctas_and_sm_capped_grids():
    """The shapes above do what they claim: a partial last CTA for every C, and a reduce grid capped by num_sms."""
    sms = 132
    for C in CS:
        M = _ms(C)[2]
        assert any(M % _plan(M, C, s, True)[0] for s in (1, 3, 7, sms, 1000)), C
        if C < 4096:
            assert M % _rgroups(C), C
    assert _plan(131072, 64, sms, True) == (1024, 128)
    assert _plan(131072, 64, 1000, True)[1] == 512


def _lib():
    from draco_b200.ops import norm
    return norm._lib()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ck(rc, what):
    from draco_b200 import _native as N
    N.check(rc, what)


def _p(t):
    return None if t is None else t.data_ptr()


def _gen(*seed):
    g = torch.Generator()
    g.manual_seed(zlib.crc32(repr(seed).encode()))
    return g


def _dev(*ts):
    return [None if t is None else t.to(DEV) for t in ts]


def _check(out, ref, what):
    """Bit-for-bit by value (+0 == -0, NaN == NaN); the message names the first differing (row, channel) or channel."""
    a, b = out.float(), ref.to(out.device).float()
    if torch.equal(a, b) or not bool(((a != b) & ~(a.isnan() & b.isnan())).any()):
        return
    X.assert_equal(out, ref.to(out.device), what + (" [index (row, channel)]" if out.dim() == 2 else ""))


def _garbage(shape, dtype):
    """Output buffers start as a value no kernel writes, so an element left unwritten is seen."""
    if dtype == torch.uint8:
        return torch.full(shape, 0x5A, dtype=dtype, device=DEV)
    return torch.full(shape, -12345.0, dtype=dtype, device=DEV)


def _specials(t, k0):
    """Sprinkle +-0, NaN and +-Inf into a flat view (real-data cases)."""
    f = t.view(-1)
    f[k0::13] = 0.0
    f[k0 + 1::13] = -0.0
    f[k0 + 3::17] = float("nan")
    f[k0 + 4::19] = float("inf")
    f[k0 + 5::23] = float("-inf")
    return t


def _real_params(C, g):
    """gamma, beta, mean, invstd: every fourth channel has gamma = 2^-20, beta = mean = 0 and invstd = 1, so inputs of 2^-126
    give fp32 outputs that are positive but round to bf16 zero."""
    gamma = torch.rand(C, generator=g) + 0.5
    beta = torch.rand(C, generator=g) - 0.5
    mean = torch.randn(C, generator=g) * 0.3
    invstd = torch.rand(C, generator=g) + 0.3
    tiny = torch.arange(C) % 4 == 0
    gamma[tiny], beta[tiny], mean[tiny], invstd[tiny] = 2.0 ** -20, 0.0, 0.0, 1.0
    return gamma, beta, mean, invstd


def _real_act(M, C, g, k0):
    x = torch.randn(M, C, generator=g) * 1.5 + 0.2
    x.view(-1)[k0 + 2::11] = 2.0 ** -126
    return _specials(x, k0).to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------------------------------------
# forward apply
# ------------------------------------------------------------------------------------------------------------------------------
def _fwd(x, res, gamma, beta, mean, invstd, relu, sms, have_stats=1, ws=None, counter=None):
    M, C = x.shape
    y = _garbage((M, C), torch.bfloat16)
    mask = _garbage((M * C // 8,), torch.uint8)
    _ck(_lib().drc_bn_fwd(x.data_ptr(), _p(res), y.data_ptr(), mask.data_ptr(), gamma.data_ptr(), beta.data_ptr(), None, None,
                          mean.data_ptr(), invstd.data_ptr(), _p(ws), _p(counter), M, C, 1e-5, 0.1, int(relu), sms,
                          have_stats, _stream()), "bn_fwd")
    return y, mask


def test_unsupported_channel_counts_are_refused():
    lib = _lib()
    for C in (4, 12, 24, 40, 8192):
        assert lib.drc_bn_supported(C) == 0 and lib.drc_bn_workspace(64, C, 132) == -1, C
    for C in CS:
        assert lib.drc_bn_supported(C) == 1, C


@pytest.mark.parametrize("M,C", SHAPES)
def test_bn_forward_apply_exact(M, C):
    """bn_apply_kernel<false> with and without residual and ReLU: y and the ReLU bits equal bn_apply_ref for every grid plan;
    with have_stats = 0 the apply uses the statistics kernel's mean / invstd exactly as the reference does."""
    g = _gen("fwd", M, C)
    x = _real_act(M, C, g, 0)
    res = _specials(torch.randn(M, C, generator=g), 6).to(torch.bfloat16)
    prm = _real_params(C, g)
    xd, rd, *prmd = _dev(x, res, *prm)
    for with_res in (False, True):
        for relu in (False, True):
            y_ref, keep = X.bn_apply_ref(x, res if with_res else None, *prm, relu)
            y_ref, keep = y_ref.to(DEV), keep.to(DEV)
            for sms in _sms_list():
                y, mask = _fwd(xd, rd if with_res else None, *prmd, relu, sms)
                what = f"M={M} C={C} res={with_res} relu={relu} num_sms={sms}"
                _check(y, y_ref, "y " + what)
                if relu:
                    _check(X.unpack_relu_bits(mask, (M, C)), keep, "mask " + what)
    # statistics computed by the forward itself (finite data: the statistics kernel is tested in test_exact_kernels_gpu.py)
    xc = (torch.randn(M, C, generator=g) * 1.5 + 0.2).to(torch.bfloat16)
    sms = _sms_list()[3]
    mean, invstd = torch.empty(C, device=DEV), torch.empty(C, device=DEV)
    ws = torch.empty(int(_lib().drc_bn_workspace(M, C, sms)), device=DEV)
    counter = torch.zeros(1, dtype=torch.int32, device=DEV)
    y, mask = _fwd(xc.to(DEV), rd, prmd[0], prmd[1], mean, invstd, True, sms, 0, ws, counter)
    y_ref, keep = X.bn_apply_ref(xc, res, prm[0], prm[1], mean, invstd, True)
    _check(y, y_ref, "y (have_stats = 0)")
    _check(X.unpack_relu_bits(mask, (M, C)), keep, "mask (have_stats = 0)")
    assert int(counter[0]) == 0


@pytest.mark.parametrize("M,C", SHAPES)
def test_bn_pair_forward_exact(M, C):
    """bn_apply_kernel<true> (drc_bn_fwd_dual): relu(bn(x) + bf16(bn_s(xs))), including C = 4096 (64 KB of coefficients)."""
    g = _gen("pair", M, C)
    x = _real_act(M, C, g, 0)
    xs = _real_act(M, C, g, 7)
    prm = _real_params(C, g)
    prm_s = _real_params(C, g)
    y_ref, keep = X.bn_apply_ref(x, None, *prm, True, pair=(xs, *prm_s))
    xd, xsd, *pd = _dev(x, xs, *prm, *prm_s)
    for sms in _sms_list():
        y = _garbage((M, C), torch.bfloat16)
        mask = _garbage((M * C // 8,), torch.uint8)
        _ck(_lib().drc_bn_fwd_dual(xd.data_ptr(), xsd.data_ptr(), y.data_ptr(), mask.data_ptr(), *(t.data_ptr() for t in pd),
                                   M, C, sms, _stream()), "bn_fwd_dual")
        _check(y, y_ref, f"pair y M={M} C={C} num_sms={sms}")
        _check(X.unpack_relu_bits(mask, (M, C)), keep.to(DEV), f"pair mask M={M} C={C} num_sms={sms}")


# ------------------------------------------------------------------------------------------------------------------------------
# backward: reduce (exact on integer data) and apply
# ------------------------------------------------------------------------------------------------------------------------------
def _bwd(dy, y, mask, x, gamma, beta, mean, invstd, mode, with_dres, sms, counter):
    M, C = x.shape
    dx = _garbage((M, C), torch.bfloat16)
    dres = _garbage((M, C), torch.bfloat16) if with_dres else None
    dgamma, dbeta, sums = _garbage((C,), torch.float32), _garbage((C,), torch.float32), _garbage((2 * C,), torch.float32)
    ws = torch.empty(int(_lib().drc_bn_workspace(M, C, sms)), device=DEV)
    _ck(_lib().drc_bn_bwd(dy.data_ptr(), _p(y if mode == 1 else None), _p(mask if mode == 3 else None), x.data_ptr(),
                          gamma.data_ptr(), _p(beta if mode == 2 else None), mean.data_ptr(), invstd.data_ptr(), dx.data_ptr(),
                          _p(dres), dgamma.data_ptr(), dbeta.data_ptr(), ws.data_ptr(), sums.data_ptr(), counter.data_ptr(),
                          M, C, mode, sms, _stream()), "bn_bwd")
    return dx, dres, dgamma, dbeta, sums


def _bwd_dual(dy, mask, x, xs, gamma, mean, invstd, gamma_s, mean_s, invstd_s, sms, counter):
    M, C = x.shape
    dx, dxs = _garbage((M, C), torch.bfloat16), _garbage((M, C), torch.bfloat16)
    dg, db, dgs, dbs = (_garbage((C,), torch.float32) for _ in range(4))
    sums, sums_s = _garbage((2 * C,), torch.float32), _garbage((2 * C,), torch.float32)
    ws = torch.empty(int(_lib().drc_bn_workspace(M, C, sms)) // 2 * 3, device=DEV)
    _ck(_lib().drc_bn_bwd_dual(dy.data_ptr(), mask.data_ptr(), x.data_ptr(), xs.data_ptr(), gamma.data_ptr(), mean.data_ptr(),
                               invstd.data_ptr(), gamma_s.data_ptr(), mean_s.data_ptr(), invstd_s.data_ptr(), dx.data_ptr(),
                               dxs.data_ptr(), dg.data_ptr(), db.data_ptr(), dgs.data_ptr(), dbs.data_ptr(), ws.data_ptr(),
                               sums.data_ptr(), sums_s.data_ptr(), counter.data_ptr(), M, C, sms, _stream()), "bn_bwd_dual")
    return dx, dxs, dg, db, dgs, dbs, sums, sums_s


def _int_case(M, C, g):
    x = torch.randint(-8, 9, (M, C), generator=g).to(torch.bfloat16)
    xs = torch.randint(-8, 9, (M, C), generator=g).to(torch.bfloat16)
    dy = torch.randint(-1, 2, (M, C), generator=g).to(torch.bfloat16)
    gamma, beta, gamma_s = torch.rand(C, generator=g) + 0.5, torch.rand(C, generator=g) - 0.5, torch.rand(C, generator=g) + 0.5
    mean, mean_s = (torch.randint(-3, 4, (C,), generator=g).float() for _ in range(2))
    q = torch.full((C,), 0.25)
    return x, xs, dy, gamma, beta, gamma_s, mean, mean_s, q


@pytest.mark.parametrize("M,C", SHAPES)
def test_bn_backward_reduce_exact(M, C):
    """Mask modes 0-3 with and without dres, and the downsampling pair's dual reduce, on integer data: dgamma, dbeta, both
    sums rows (and the pair's dgamma_s, dbeta_s, sums_s) exact; dres = bf16(dz); dx / dxs equal bn_bwd_apply_ref of those sums.
    Every case runs twice on one counter (the last CTA resets the ticket): both launches give the reference bits."""
    g = _gen("reduce", M, C)
    x, xs, dy, gamma, beta, gamma_s, mean, mean_s, q = _int_case(M, C, g)
    xd, xsd, dyd, gd, bd, gsd, md, msd, qd = _dev(x, xs, dy, gamma, beta, gamma_s, mean, mean_s, q)
    # the forward's outputs for modes 1 and 3; mode 2 recomputes the same mask from x (no residual)
    y_ref, keep = X.bn_apply_ref(x, None, gamma, beta, mean, q, True)
    y, mask = _fwd(xd, None, gd, bd, md, qd, True, _sms_list()[3])
    _check(y, y_ref, "forward y")
    assert 0 < int(keep.sum()) < keep.numel() or M == 1
    counter = torch.zeros(1, dtype=torch.int32, device=DEV)
    for mode in (0, 1, 2, 3):
        k = None if mode == 0 else keep
        dz = dy if k is None else torch.where(k, dy, torch.zeros_like(dy))
        dbeta, dgamma, sums = X.bn_bwd_sums_ref(dz, x, mean, q)
        X.assert_exact_domain(4 * (dz.double() * (x.double() - mean) * 0.25).abs().sum(0))      # partial sums on a 1/4 grid
        dx_ref, dres_ref = X.bn_bwd_apply_ref(dy, k, x, X.bn_bwd_coeffs_ref(gamma, q, mean, sums))
        refs = _dev(dx_ref, dres_ref, dgamma.float(), dbeta.float(), sums)
        for with_dres in (False, True):
            for sms in _sms_list():
                for launch in (1, 2):
                    dx, dres, dg, db, s = _bwd(dyd, y, mask, xd, gd, bd, md, qd, mode, with_dres, sms, counter)
                    what = f"mode={mode} dres={with_dres} M={M} C={C} num_sms={sms} launch {launch}"
                    _check(dg, refs[2], "dgamma [channel] " + what)
                    _check(db, refs[3], "dbeta [channel] " + what)
                    _check(s, refs[4], "sums [row * C + channel] " + what)
                    _check(dx, refs[0], "dx " + what)
                    if with_dres:
                        _check(dres, refs[1], "dres " + what)
                    assert int(counter[0]) == 0, "ticket not reset: " + what
    # downsampling pair: one reduce for both layers
    dz = torch.where(keep, dy, torch.zeros_like(dy))
    dbeta, dgamma, sums = X.bn_bwd_sums_ref(dz, x, mean, q)
    _, dgamma_s, sums_s = X.bn_bwd_sums_ref(dz, xs, mean_s, q)
    dx_ref, _ = X.bn_bwd_apply_ref(dy, keep, x, X.bn_bwd_coeffs_ref(gamma, q, mean, sums))
    dxs_ref, _ = X.bn_bwd_apply_ref(dy, keep, xs, X.bn_bwd_coeffs_ref(gamma_s, q, mean_s, sums_s))
    refs = _dev(dx_ref, dxs_ref, dgamma.float(), dbeta.float(), dgamma_s.float(), dbeta.float(), sums, sums_s)
    names = ["dx", "dxs", "dgamma [channel]", "dbeta [channel]", "dgamma_s [channel]", "dbeta_s [channel]",
             "sums [row * C + channel]", "sums_s [row * C + channel]"]
    for sms in _sms_list():
        for launch in (1, 2):
            out = _bwd_dual(dyd, mask, xd, xsd, gd, md, qd, gsd, msd, qd, sms, counter)
            for o, r, n in zip(out, refs, names):
                _check(o, r, f"pair {n} M={M} C={C} num_sms={sms} launch {launch}")
            assert int(counter[0]) == 0


@pytest.mark.parametrize("M,C", SHAPES)
def test_bn_backward_apply_exact_on_real_data(M, C):
    """Real-valued data: for every mask mode (with dres) and the pair, dx, dres and dxs equal bn_bwd_apply_ref of the sums the
    launch itself produced, the sums rows are rn32(dbeta * rn32(1/M)) and rn32(dgamma * rn32(1/M)) of the kernel's own dbeta
    and dgamma, and the reduction is within |dgamma - ref64| <= (M + 2) 2^-23 sum |dz| |xhat| (xhat rounded twice in fp32,
    fma-accumulated), |dbeta - ref64| <= (M + 1) 2^-23 sum |dz|."""
    g = _gen("real", M, C)
    x = (torch.randn(M, C, generator=g) * 1.7 + torch.randn(C, generator=g)).to(torch.bfloat16)
    xs = (torch.randn(M, C, generator=g) * 0.9 - 0.3).to(torch.bfloat16)
    dy = torch.randn(M, C, generator=g).to(torch.bfloat16)
    gamma, beta, gamma_s = torch.rand(C, generator=g) + 0.5, torch.rand(C, generator=g) - 0.5, torch.rand(C, generator=g) + 0.5
    mean, mean_s = x.float().mean(0), xs.float().mean(0)
    invstd, invstd_s = (x.float().var(0, unbiased=False) + 1e-5).rsqrt(), (xs.float().var(0, unbiased=False) + 1e-5).rsqrt()
    xd, xsd, dyd, gd, bd, gsd, md, msd, isd, iss = _dev(x, xs, dy, gamma, beta, gamma_s, mean, mean_s, invstd, invstd_s)
    _, keep = X.bn_apply_ref(x, None, gamma, beta, mean, invstd, True)
    y, mask = _fwd(xd, None, gd, bd, md, isd, True, _sms_list()[3])
    inv_m = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(float(M), dtype=torch.float32)
    xhat = (x.double() - mean.double()) * invstd.double()

    def check_sums(dg, db, s, dz, what):
        dg, db, s = dg.cpu(), db.cpu(), s.cpu()
        X.assert_equal(s, torch.cat([db * inv_m, dg * inv_m]), "sums of the kernel's dbeta, dgamma " + what)
        dzd = dz.double()
        assert bool(((db.double() - dzd.sum(0)).abs() <= (M + 1) * 2.0 ** -23 * dzd.abs().sum(0)).all()), "dbeta " + what
        X.assert_bound(dg, (dzd * xhat).sum(0), (dzd * xhat).abs().sum(0), M + 2, "dgamma " + what, rel=0.0)

    counter = torch.zeros(1, dtype=torch.int32, device=DEV)
    for mode in (0, 1, 2, 3):
        k = None if mode == 0 else keep
        dz = dy if k is None else torch.where(k, dy, torch.zeros_like(dy))
        for sms in (1, _sms_list()[3]):
            what = f"mode={mode} M={M} C={C} num_sms={sms}"
            dx, dres, dg, db, s = _bwd(dyd, y, mask, xd, gd, bd, md, isd, mode, True, sms, counter)
            dx_ref, dres_ref = X.bn_bwd_apply_ref(dy, k, x, X.bn_bwd_coeffs_ref(gamma, invstd, mean, s))
            _check(dx, dx_ref, "dx " + what)
            _check(dres, dres_ref, "dres " + what)
            check_sums(dg, db, s, dz, what)
    dz = torch.where(keep, dy, torch.zeros_like(dy))
    for sms in (1, _sms_list()[3]):
        what = f"pair M={M} C={C} num_sms={sms}"
        dx, dxs, dg, db, dgs, dbs, s, ss = _bwd_dual(dyd, mask, xd, xsd, gd, md, isd, gsd, msd, iss, sms, counter)
        _check(dx, X.bn_bwd_apply_ref(dy, keep, x, X.bn_bwd_coeffs_ref(gamma, invstd, mean, s))[0], "dx " + what)
        _check(dxs, X.bn_bwd_apply_ref(dy, keep, xs, X.bn_bwd_coeffs_ref(gamma_s, invstd_s, mean_s, ss))[0], "dxs " + what)
        _check(dbs, db, "dbeta_s [channel] " + what)
        _check(ss[:C], s[:C], "sums_s[0] [channel] " + what)
        check_sums(dg, db, s, dz, what)
        X.assert_equal(ss[C:].cpu(), dgs.cpu() * inv_m, "sums_s[1] [channel] " + what)


@pytest.mark.parametrize("M,C", SHAPES)
def test_bn_apply_only_exact(M, C):
    """drc_bn_bwd_apply (the apply after a dgrad epilogue reduced the sums): dx from given real sums, with +-0, NaN and +-Inf in
    dz and x, equals bn_bwd_apply_ref element by element."""
    g = _gen("apply", M, C)
    dz = _specials(torch.randn(M, C, generator=g), 0).to(torch.bfloat16)
    x = _real_act(M, C, g, 5)
    gamma, _, mean, invstd = _real_params(C, g)
    sums = torch.randn(2 * C, generator=g) * 0.2
    sums[:C:5] = 0.0
    dx_ref, _ = X.bn_bwd_apply_ref(dz, None, x, X.bn_bwd_coeffs_ref(gamma, invstd, mean, sums))
    dzd, xd, gd, md, isd, sd = _dev(dz, x, gamma, mean, invstd, sums)
    for sms in _sms_list():
        dx = _garbage((M, C), torch.bfloat16)
        _ck(_lib().drc_bn_bwd_apply(dzd.data_ptr(), xd.data_ptr(), gd.data_ptr(), md.data_ptr(), isd.data_ptr(), sd.data_ptr(),
                                    dx.data_ptr(), M, C, sms, _stream()), "bn_bwd_apply")
        _check(dx, dx_ref, f"apply-only dx M={M} C={C} num_sms={sms}")


# ------------------------------------------------------------------------------------------------------------------------------
# the autograd ops the model runs: _BnActFn (every DRACO_BN_MASK) and _BnPairFn
# ------------------------------------------------------------------------------------------------------------------------------
def _rows(t):
    """NCHW (channels-last) -> [M, C] pixel rows."""
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])


@pytest.mark.parametrize("op", ["bits+res", "y+res", "x", "bits", "no-relu+res", "pair"])
def test_fused_batchnorm_autograd_exact(op, monkeypatch):
    """FusedBatchNorm2d with statistics handed over as pending_stats (integer means, invstd = 1/4, integer data): y, dx,
    dres / dxs, dgamma and dbeta equal the references bit for bit."""
    from draco_b200.ops import norm
    n, c, h, w = 5, 64, 7, 9
    monkeypatch.setenv("DRACO_BN_MASK", op.split("+")[0] if op[0] in "bxy" else "bits")
    g = _gen("autograd", op)
    M = n * h * w
    x, xs, dy, gamma, beta, gamma_s, mean, mean_s, q = _int_case(M, c, g)
    beta_s = torch.rand(c, generator=g) - 0.5
    relu = not op.startswith("no-relu")
    with_res = op.endswith("+res")
    res = torch.randint(-4, 5, (M, c), generator=g).to(torch.bfloat16) if with_res else None

    def nchw(t):
        return t.to(DEV).reshape(n, h, w, c).permute(0, 3, 1, 2)

    bns = []
    for gm, bt in ((gamma, beta), (gamma_s, beta_s)):
        bn = norm.FusedBatchNorm2d(c).to(DEV)
        with torch.no_grad():
            bn.weight.copy_(gm)
            bn.bias.copy_(bt)
        bns.append(bn)
    bn, bn_s = bns
    xg, sg = nchw(x).requires_grad_(True), nchw(xs).requires_grad_(True)
    rg = nchw(res).requires_grad_(True) if with_res else None
    bn.pending_stats = (xg, mean.to(DEV), q.to(DEV))
    before = norm.backend_counters["fused"]
    if op == "pair":
        bn_s.pending_stats = (sg, mean_s.to(DEV), q.to(DEV))
        y = bn(xg, residual_bn=(bn_s, sg), relu=True)
        assert norm.backend_counters["fused"] - before == 2
        y_ref, keep = X.bn_apply_ref(x, None, gamma, beta, mean, q, True, pair=(xs, gamma_s, beta_s, mean_s, q))
    else:
        y = bn(xg, residual=rg, relu=relu)
        assert norm.backend_counters["fused"] - before == 1
        y_ref, keep = X.bn_apply_ref(x, res, gamma, beta, mean, q, relu)
    y.backward(nchw(dy))
    torch.cuda.synchronize()
    _check(_rows(y.detach()), y_ref, f"{op}: y")
    k = keep if relu else None
    dz = dy if k is None else torch.where(k, dy, torch.zeros_like(dy))
    dbeta, dgamma, sums = X.bn_bwd_sums_ref(dz, x, mean, q)
    dx_ref, dres_ref = X.bn_bwd_apply_ref(dy, k, x, X.bn_bwd_coeffs_ref(gamma, q, mean, sums))
    _check(_rows(xg.grad), dx_ref, f"{op}: dx")
    _check(bn.weight.grad, dgamma.float(), f"{op}: dgamma [channel]")
    _check(bn.bias.grad, dbeta.float(), f"{op}: dbeta [channel]")
    if with_res:
        _check(_rows(rg.grad), dres_ref, f"{op}: dres")
    if op == "pair":
        _, dgamma_s, sums_s = X.bn_bwd_sums_ref(dz, xs, mean_s, q)
        dxs_ref, _ = X.bn_bwd_apply_ref(dy, keep, xs, X.bn_bwd_coeffs_ref(gamma_s, q, mean_s, sums_s))
        _check(_rows(sg.grad), dxs_ref, f"{op}: dxs")
        _check(bn_s.weight.grad, dgamma_s.float(), f"{op}: dgamma_s [channel]")
        _check(bn_s.bias.grad, dbeta.float(), f"{op}: dbeta_s [channel]")
