"""Exact tests of the tensor-core GEMM, the convolution families, the BatchNorm statistics they produce and the head kernels.

Operands are small integers ({-1, 0, +1}, see tests/exact_ref.py), so every product and every fp32 partial sum is exact in any
summation order: a bf16 output has to equal the fp64 reference rounded once to nearest-even BIT FOR BIT, whatever the tile
shape, split-K plan, cluster shape or epilogue.  Integer offsets (a bias of +-(1000 + k), residuals of |r| <= 300) push outputs
past 256, where bf16 has to round and ties occur: they pin round-to-nearest-even.  One real-valued case per entry point checks
the per-element bound |y - ref64| <= 2^-8 |ref64| + (K + 1) 2^-23 (|x| (*) |w|) (derived in exact_ref.py).

Shapes are non-square (H < W and H > W), have odd output sizes and 1-pixel outputs, channel counts 192 / 320 / 448 (an odd number
of 64-wide K blocks, partial 128-wide N tiles) and 576 / 640, batches that leave the last pixel tile partial, and ImageNet sizes.
"""
import os

import pytest
import torch

import exact_ref as X

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)

CLUSTER_CFGS = ["2,1,128", "1,2,128", "2,2,128", "4,2,128", "2,4,64", "8,1,64", "1,8,64", "4,1,128", "1,4,64", "2,1,64", "1,2,64",
                "2,2,64", "4,2,64", "1,1,64", "1,1,128"]


@pytest.fixture(autouse=True)
def _no_tf32():
    m, c = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = m, c


def _gen(seed):
    g = torch.Generator()
    g.manual_seed(seed)
    return g


def _iop(shape, K, g, target=2 ** 11):
    return X.int_operand(shape, K, g, target, DEV)


def _offset_bias(c):
    """fp32 bias of +-(1000 + k): every output needs rounding to bf16 (spacing 4 or 8 there), many land on ties."""
    k = torch.arange(c, device=DEV)
    return ((1000 + (k * 7) % 61) * (1 - 2 * (k % 2))).float()


def _sms():
    from draco_b200.ops import kernels as K
    return K.sm_count(DEV)


# ------------------------------------------------------------------------------------------------------------------------------
# GEMM (csrc/cuda/gemm_wgmma.cu)
# ------------------------------------------------------------------------------------------------------------------------------
GEMM_SHAPES = [(128, 128, 64), (77, 136, 72), (200, 10, 512), (300, 504, 784), (130, 264, 1032), (1000, 16, 512), (64, 64, 8),
               (515, 328, 1000), (136, 40, 4608)]


@pytest.mark.parametrize("M,N,Kd", GEMM_SHAPES)
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, False), (True, True)])
def test_gemm_exact_operand_orders(M, N, Kd, a_mn, b_mn):
    from draco_b200.ops import kernels as K
    if (a_mn and M % 8) or (b_mn and N % 8):
        pytest.skip("an MN-major operand needs a 16-byte row pitch")
    g = _gen(M * 7 + N * 3 + Kd)
    A, B = _iop((M, Kd), Kd, g), _iop((N, Kd), Kd, g)
    ref = A.double() @ B.double().t()
    A16, B16 = A.to(torch.bfloat16), B.to(torch.bfloat16)
    A_in = A16.t().contiguous() if a_mn else A16
    B_in = B16.t().contiguous() if b_mn else B16
    X.assert_equal(K.gemm_bf16(A_in, B_in, a_mn=a_mn, b_mn=b_mn, out_dtype=torch.float32), ref.float(), "fp32 out")
    X.assert_equal(K.gemm_bf16(A_in, B_in, a_mn=a_mn, b_mn=b_mn), X.bf16_rn(ref), "bf16 out")
    bias = _offset_bias(N)
    X.assert_equal(K.gemm_bf16(A_in, B_in, a_mn=a_mn, b_mn=b_mn, bias=bias), X.bf16_rn(ref + bias.double()), "bf16 out + bias")


@pytest.mark.parametrize("block_n", [32, 64, 128, 256])
@pytest.mark.parametrize("M,N,Kd", [(515, 328, 1000), (200, 10, 72), (131, 72, 136)])
def test_gemm_exact_block_n_bias_relu_accumulate(block_n, M, N, Kd):
    from draco_b200.ops import kernels as K
    g = _gen(block_n + M)
    A, B = _iop((M, Kd), Kd, g), _iop((N, Kd), Kd, g)
    ref = A.double() @ B.double().t()
    A16, B16 = A.to(torch.bfloat16), B.to(torch.bfloat16)
    bias = _offset_bias(N)
    refb = ref + bias.double()
    run = lambda **kw: K.gemm_bf16(A16, B16, block_n=block_n, **kw)      # noqa: E731
    X.assert_equal(run(out_dtype=torch.float32, bias=bias), refb.float(), "fp32 + bias")
    X.assert_equal(run(bias=bias), X.bf16_rn(refb), "bf16 + bias")
    X.assert_equal(run(bias=bias, relu=True), X.bf16_rn(refb.clamp_min(0)), "bf16 + bias + relu")
    X.assert_equal(run(out_dtype=torch.float32, bias=bias, relu=True), refb.clamp_min(0).float(), "fp32 + bias + relu")
    b16 = X.bf16_rn(bias.double() * 0.3)                                  # bf16 bias: +-(300..318), representable after rounding
    X.assert_equal(run(bias=b16), X.bf16_rn(ref + b16.double()), "bf16 + bf16 bias")
    acc0 = torch.randint(-3000, 3000, (M, N), generator=g).float().to(DEV)
    acc = acc0.clone()
    run(out=acc, accumulate=True)
    X.assert_equal(acc, (acc0.double() + ref).float(), "fp32 accumulate")
    acc16_0 = (torch.randint(-150, 150, (M, N), generator=g) * 2).to(torch.bfloat16).to(DEV)
    acc16 = acc16_0.clone()
    run(out=acc16, accumulate=True)
    X.assert_equal(acc16, X.bf16_rn(acc16_0.double() + ref), "bf16 accumulate (one rounding of the exact sum)")
    if block_n >= 64 and N % 8 == 0:                                      # MN-major B: the tile is at least 64 wide
        Bt = B16.t().contiguous()
        X.assert_equal(K.gemm_bf16(A16, Bt, b_mn=True, block_n=block_n, bias=bias), X.bf16_rn(refb), "b_mn + bias")


@pytest.mark.parametrize("M,N,Kd", [(200, 10, 72), (130, 264, 1032), (77, 40, 512)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("col0", [8, 3])
def test_gemm_out_view_leaves_guard_cells_untouched(M, N, Kd, dtype, col0):
    """``out=`` a view into a larger sentinel-filled buffer (16-byte aligned view: vector stores; col0 = 3: scalar stores):
    the view holds the exact result, every row and column around it keeps the sentinel."""
    from draco_b200.ops import kernels as K
    g = _gen(M + N + col0)
    A, B = _iop((M, Kd), Kd, g), _iop((N, Kd), Kd, g)
    ref = A.double() @ B.double().t()
    sentinel = -12345.0 if dtype == torch.float32 else float(torch.tensor(-12352.0).to(torch.bfloat16))
    big = torch.full((M + 5, N + 24), sentinel, dtype=dtype, device=DEV)
    out = big[2:2 + M, col0:col0 + N]
    K.gemm_bf16(A.to(torch.bfloat16), B.to(torch.bfloat16), out=out, out_dtype=dtype)
    exp = ref.float() if dtype == torch.float32 else X.bf16_rn(ref)
    X.assert_equal(out, exp, "view")
    guard = torch.ones_like(big, dtype=torch.bool)
    guard[2:2 + M, col0:col0 + N] = False
    assert bool((big[guard] == sentinel).all()), "the GEMM wrote outside its output view"
    K.gemm_bf16(A.to(torch.bfloat16), B.to(torch.bfloat16), out=out, accumulate=True)
    exp2 = (2 * ref).float() if dtype == torch.float32 else X.bf16_rn(X.bf16_rn(ref).double() + ref)
    X.assert_equal(out, exp2, "view, accumulate")
    assert bool((big[guard] == sentinel).all()), "the accumulating GEMM wrote outside its output view"


def test_gemm_randn_component_bound():
    from draco_b200.ops import kernels as K
    g = _gen(5)
    for M, N, Kd in [(300, 504, 784), (200, 10, 4608)]:
        A = torch.randn(M, Kd, generator=g).to(torch.bfloat16).to(DEV)
        B = torch.randn(N, Kd, generator=g).to(torch.bfloat16).to(DEV)
        ref = A.double() @ B.double().t()
        aref = A.double().abs() @ B.double().abs().t()
        X.assert_bound(K.gemm_bf16(A, B, out_dtype=torch.float32), ref, aref, Kd, "fp32 out", rel=2.0 ** -24)
        X.assert_bound(K.gemm_bf16(A, B), ref, aref, Kd, "bf16 out")
        a_mn, b_mn = M % 8 == 0, N % 8 == 0                                   # MN-major operands need a 16-byte row pitch
        out = K.gemm_bf16(A.t().contiguous() if a_mn else A, B.t().contiguous() if b_mn else B, a_mn=a_mn, b_mn=b_mn)
        X.assert_bound(out, ref, aref, Kd, "MN-major")


# ------------------------------------------------------------------------------------------------------------------------------
# tap-table convolutions (csrc/cuda/conv_tap_wgmma.cu): every epilogue, tile width and cluster shape against one reference
# ------------------------------------------------------------------------------------------------------------------------------
# (n, cin, cout, H, W, ks, stride)
TAP_CASES = [
    (5, 192, 320, 4, 8, 3, 1),      # H < W; patch 8 x 4 x 4 images: the second tile holds 1 of 4; 3 K blocks per tap; 320 = 2.5 tiles
    (3, 320, 192, 16, 4, 3, 1),     # H > W; patch 4 x 16 x 2 images, N odd; Cin 320 = 5 K blocks
    (4, 448, 448, 6, 14, 3, 2),     # OH = 3, OW = 7 (odd): 1 x 1 x 128 patches, 4 of 128 images valid; parity-class dgrad
    (6, 64, 576, 2, 16, 3, 2),      # OH = 1; Cout 576 (no statistics)
    (3, 128, 640, 14, 1, 3, 1),     # OW = 1; Cout 640
    (5, 192, 320, 8, 12, 1, 2),     # 1x1 / stride 2: dgrad classes without taps are zeroed by the memset
    (7, 320, 448, 8, 4, 1, 1),      # 1x1 / stride 1, H > W
    (2, 64, 128, 56, 56, 3, 2),     # ImageNet: 56 -> 28 downsampling
    (3, 128, 128, 28, 28, 3, 1),    # ImageNet: 28 x 28
]


def _variants(n, cin, cout, h, w, ks, stride, dgrad):
    """(DRACO_CONV_EPI, DRACO_CONV_CLUSTER) pairs the launcher realises for this layer: both epilogues of the default plan, then
    every forced tile width / cluster shape the planner accepts (the stride-2 dgrad always uses the direct epilogue)."""
    from draco_b200.ops.conv import convg_plan
    out = [("tma", None), ("direct", None)]
    sms = _sms()
    for cfg in CLUSTER_CFGS:
        os.environ["DRACO_CONV_CLUSTER"] = cfg
        try:
            plan = convg_plan(n, h, w, cin, cout, ks, stride, dgrad, sms)
        finally:
            del os.environ["DRACO_CONV_CLUSTER"]
        cm, cn, bn = (int(v) for v in cfg.split(","))
        if plan is not None and plan[:3] == [bn, cm, cn] and plan[4] == (1 if cm * cn > 1 else 0):
            out.append(("tma", cfg))
    return out


def _set_variant(monkeypatch, epi, cfg):
    monkeypatch.setenv("DRACO_CONV_EPI", epi)
    if cfg is None:
        monkeypatch.delenv("DRACO_CONV_CLUSTER", raising=False)
    else:
        monkeypatch.setenv("DRACO_CONV_CLUSTER", cfg)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("n,cin,cout,h,w,ks,stride", TAP_CASES)
def test_convg_tap_exact_every_variant(n, cin, cout, h, w, ks, stride, monkeypatch):
    from draco_b200.ops.conv import convg_tcgen05, convg_wgrad_tcgen05
    g = _gen(n + cin + cout + h + 3 * w + ks + stride)
    oh, ow = h // stride, w // stride
    x = _iop((n, cin, h, w), ks * ks * cin, g)
    wt = _iop((cout, cin, ks, ks), ks * ks * cin, g)
    dy = _iop((n, cout, oh, ow), ks * ks * cout, g)
    bias = _offset_bias(cout)
    b16 = X.bf16_rn(bias.double() * 0.3)
    res = (torch.randint(-150, 151, (n, cin, h, w), generator=g) * 2).float().to(DEV)     # even, |r| <= 300: exact in bf16
    xb, wb, dyb, rb = X.cl(x), X.wt(wt), X.cl(dy), X.cl(res)
    y64 = X.conv_ref(x, wt, stride)
    dx64 = X.dgrad_ref(dy, wt, (h, w), stride)
    X.assert_exact_domain(y64, dx64)
    ref_y = X.bf16_rn(y64 + bias.double().view(1, -1, 1, 1))
    ref_yb = X.bf16_rn(y64 + b16.double().view(1, -1, 1, 1))
    ref_dx = X.bf16_rn(dx64)
    ref_dxr = X.bf16_rn(dx64 + res.double())
    with_res = not (ks == 1 and stride == 2)
    fvars, dvars = _variants(n, cin, cout, h, w, ks, stride, 0), _variants(n, cin, cout, h, w, ks, stride, 1)
    ran = []
    for epi, cfg in fvars:
        _set_variant(monkeypatch, epi, cfg)
        y = convg_tcgen05(xb, wb, (h, w), stride, False, bias)
        assert y.is_contiguous(memory_format=torch.channels_last)
        X.assert_equal(y, ref_y, f"fprop + fp32 bias [{epi}, {cfg}]")
        X.assert_equal(convg_tcgen05(xb, wb, (h, w), stride, False, b16), ref_yb, f"fprop + bf16 bias [{epi}, {cfg}]")
        ran.append(("fprop", epi, cfg))
    for epi, cfg in dvars:
        _set_variant(monkeypatch, epi, cfg)
        X.assert_equal(convg_tcgen05(dyb, wb, (h, w), stride, True), ref_dx, f"dgrad [{epi}, {cfg}]")
        if with_res:
            X.assert_equal(convg_tcgen05(dyb, wb, (h, w), stride, True, None, None, rb), ref_dxr, f"dgrad + residual [{epi}, {cfg}]")
        ran.append(("dgrad", epi, cfg))
    _set_variant(monkeypatch, "tma", None)
    dw64 = X.wgrad_ref(dy, x, ks, stride)
    X.assert_exact_domain(dw64)
    dw = convg_wgrad_tcgen05(dyb, xb, ks, stride)
    X.assert_equal(dw, X.bf16_rn(dw64), "split-K wgrad")
    assert len(ran) >= 4


@pytest.mark.timeout(300)
@pytest.mark.parametrize("n,cin,cout,h,w,ks,stride", [TAP_CASES[0], TAP_CASES[2], TAP_CASES[5]])
def test_convg_tap_randn_component_bound(n, cin, cout, h, w, ks, stride):
    from draco_b200.ops.conv import convg_tcgen05, convg_wgrad_tcgen05
    g = _gen(n * cin + h)
    oh, ow = h // stride, w // stride
    x = torch.randn(n, cin, h, w, generator=g).to(torch.bfloat16).to(DEV)
    wt = (torch.randn(cout, cin, ks, ks, generator=g) * 0.05).to(torch.bfloat16).to(DEV)
    dy = torch.randn(n, cout, oh, ow, generator=g).to(torch.bfloat16).to(DEV)
    bias = torch.randn(cout, generator=g).to(DEV)
    y = convg_tcgen05(X.cl(x), X.wt(wt), (h, w), stride, False, bias)
    X.assert_bound(y, X.conv_ref(x, wt, stride, bias), X.conv_ref(x.abs(), wt.abs(), stride, bias.abs()), ks * ks * cin, "fprop")
    dx = convg_tcgen05(X.cl(dy), X.wt(wt), (h, w), stride, True)
    X.assert_bound(dx, X.dgrad_ref(dy, wt, (h, w), stride), X.dgrad_ref(dy.abs(), wt.abs(), (h, w), stride), ks * ks * cout, "dgrad")
    dw = convg_wgrad_tcgen05(X.cl(dy), X.cl(x), ks, stride)
    X.assert_bound(dw, X.wgrad_ref(dy, x, ks, stride), X.wgrad_ref(dy.abs(), x.abs(), ks, stride), n * oh * ow, "wgrad")


# ------------------------------------------------------------------------------------------------------------------------------
# halo-reuse kernels (csrc/cuda/conv_halo_wgmma.cu): bit-identical to the tap kernel on the same layer
# ------------------------------------------------------------------------------------------------------------------------------
HALO_CASES = [(3, 16, 64), (5, 48, 8), (1, 32, 16)]


@pytest.mark.timeout(300)
@pytest.mark.parametrize("n,h,w", HALO_CASES)
def test_conv3x3_halo_exact_equals_tap_kernel(n, h, w):
    from draco_b200.ops.conv import conv3x3_halo, conv3x3_halo_wgrad, convg_tcgen05, convg_wgrad_tcgen05, halo_supported
    assert halo_supported(h, w, 64, 64)
    g = _gen(n * h + w)
    x, wt, dy = _iop((n, 64, h, w), 576, g), _iop((64, 64, 3, 3), 576, g), _iop((n, 64, h, w), 576, g)
    bias = _offset_bias(64)
    res = (torch.randint(-150, 151, (n, 64, h, w), generator=g) * 2).float().to(DEV)
    xb, wb, dyb, rb = X.cl(x), X.wt(wt), X.cl(dy), X.cl(res)
    ref_y = X.bf16_rn(X.conv_ref(x, wt, 1, bias))
    y = conv3x3_halo(xb, wb, False, bias)
    X.assert_equal(y, ref_y, "halo fprop")
    X.assert_equal(convg_tcgen05(xb, wb, (h, w), 1, False, bias), y, "tap fprop vs halo")
    ref_dx = X.bf16_rn(X.dgrad_ref(dy, wt, (h, w), 1) + res.double())
    dx = conv3x3_halo(dyb, wb, True, None, None, rb)
    X.assert_equal(dx, ref_dx, "halo dgrad + residual")
    X.assert_equal(convg_tcgen05(dyb, wb, (h, w), 1, True, None, None, rb), dx, "tap dgrad + residual vs halo")
    X.assert_equal(conv3x3_halo(dyb, wb, True), X.bf16_rn(X.dgrad_ref(dy, wt, (h, w), 1)), "halo dgrad")
    dw = conv3x3_halo_wgrad(dyb, xb)
    X.assert_equal(dw, X.bf16_rn(X.wgrad_ref(dy, x, 3, 1)), "halo wgrad")
    X.assert_equal(convg_wgrad_tcgen05(dyb, xb, 3, 1), dw, "tap wgrad vs halo")


def test_conv3x3_halo_randn_component_bound():
    from draco_b200.ops.conv import conv3x3_halo, conv3x3_halo_wgrad
    n, h, w = 3, 16, 64
    g = _gen(17)
    x = torch.randn(n, 64, h, w, generator=g).to(torch.bfloat16).to(DEV)
    wt = (torch.randn(64, 64, 3, 3, generator=g) * 0.05).to(torch.bfloat16).to(DEV)
    dy = torch.randn(n, 64, h, w, generator=g).to(torch.bfloat16).to(DEV)
    X.assert_bound(conv3x3_halo(X.cl(x), X.wt(wt)), X.conv_ref(x, wt, 1), X.conv_ref(x.abs(), wt.abs(), 1), 576, "fprop")
    X.assert_bound(conv3x3_halo(X.cl(dy), X.wt(wt), True), X.dgrad_ref(dy, wt, (h, w), 1), X.dgrad_ref(dy.abs(), wt.abs(), (h, w), 1),
                   576, "dgrad")
    X.assert_bound(conv3x3_halo_wgrad(X.cl(dy), X.cl(x)), X.wgrad_ref(dy, x, 3, 1), X.wgrad_ref(dy.abs(), x.abs(), 3, 1), n * h * w,
                   "wgrad")


# ------------------------------------------------------------------------------------------------------------------------------
# stem (csrc/cuda/conv_stem.cu)
# ------------------------------------------------------------------------------------------------------------------------------
STEM_CASES = [(3, 16, 64), (2, 64, 8), (5, 32, 16)]


@pytest.mark.parametrize("n,h,w", STEM_CASES)
def test_conv_stem_exact(n, h, w):
    from draco_b200.ops.conv import _lib, conv_stem_fprop, conv_stem_wgrad
    assert _lib().drc_conv_stem_supported(h, w, 3, 64)
    g = _gen(n + h * w)
    x, wt = _iop((n, 3, h, w), 27, g), _iop((64, 3, 3, 3), 27, g)
    dy = _iop((n, 64, h, w), n * h * w, g)
    bias = _offset_bias(64)
    X.assert_equal(conv_stem_fprop(X.cl(x), X.wt(wt), bias), X.bf16_rn(X.conv_ref(x, wt, 1, bias)), "stem fprop")
    X.assert_equal(conv_stem_fprop(X.cl(x), X.wt(wt)), X.bf16_rn(X.conv_ref(x, wt, 1)), "stem fprop, no bias")
    X.assert_equal(conv_stem_wgrad(X.cl(dy), X.cl(x)), X.bf16_rn(X.wgrad_ref(dy, x, 3, 1)), "stem wgrad")


def test_conv_stem_randn_component_bound():
    from draco_b200.ops.conv import conv_stem_fprop, conv_stem_wgrad
    n, h, w = 3, 16, 64
    g = _gen(23)
    x = torch.randn(n, 3, h, w, generator=g).to(torch.bfloat16).to(DEV)
    wt = (torch.randn(64, 3, 3, 3, generator=g) * 0.2).to(torch.bfloat16).to(DEV)
    dy = torch.randn(n, 64, h, w, generator=g).to(torch.bfloat16).to(DEV)
    b = torch.randn(64, generator=g).to(DEV)
    X.assert_bound(conv_stem_fprop(X.cl(x), X.wt(wt), b), X.conv_ref(x, wt, 1, b), X.conv_ref(x.abs(), wt.abs(), 1, b.abs()), 27, "fprop")
    X.assert_bound(conv_stem_wgrad(X.cl(dy), X.cl(x)), X.wgrad_ref(dy, x, 3, 1), X.wgrad_ref(dy.abs(), x.abs(), 3, 1), n * h * w, "wgrad")


# ------------------------------------------------------------------------------------------------------------------------------
# BatchNorm statistics: conv epilogue (tap, halo, stem) and the standalone kernel (ops.norm) against the exact sums
# ------------------------------------------------------------------------------------------------------------------------------
def _check_stats(req, y, rm0, rv0, what):
    """mean bit-exact, invstd within 2 ulp (rsqrtf), running statistics within 1 ulp of the fp32 formula on the exact sums."""
    m, var, invstd, rm, rv = X.bn_stats_ref(y, req.eps, req.momentum, rm0, rv0)
    X.assert_equal(req.mean, m.float(), f"{what}: mean")
    assert X.ulps_f32(req.invstd, invstd) <= 2, f"{what}: invstd {X.ulps_f32(req.invstd, invstd)} ulp"
    if req.running_mean is not None:
        assert X.ulps_f32(req.running_mean, rm) <= 1, f"{what}: running_mean {X.ulps_f32(req.running_mean, rm)} ulp"
        assert X.ulps_f32(req.running_var, rv) <= 1, f"{what}: running_var {X.ulps_f32(req.running_var, rv)} ulp"


def _standalone_stats(y, eps, momentum, rm0, rv0):
    """ops.norm's statistics kernel (the DRACO_BN_STATS=kernel path) on the same tensor: mean, invstd, running statistics."""
    from draco_b200.ops.norm import FusedBatchNorm2d, backend_counters
    bn = FusedBatchNorm2d(y.shape[1], eps=eps, momentum=momentum).to(DEV)
    bn.running_mean.copy_(rm0)
    bn.running_var.copy_(rv0)
    before = backend_counters["fused"]
    out = bn(y.clone().requires_grad_(True))
    assert backend_counters["fused"] == before + 1
    link = out._draco_bn_link
    return link.mean, link.invstd, bn.running_mean, bn.running_var


# (kind, n, cin, cout, H, W, ks, stride): the last pixel tile of each is partial, so a mis-masked row changes an exact sum
STAT_CASES = [("tap", 5, 64, 128, 4, 8, 3, 1), ("tap", 3, 192, 320, 16, 4, 3, 1), ("tap", 4, 128, 256, 6, 14, 3, 2),
              ("tap", 9, 256, 512, 2, 4, 1, 1), ("halo", 3, 64, 64, 16, 64, 3, 1), ("halo", 5, 64, 64, 48, 8, 3, 1),
              ("stem", 3, 3, 64, 32, 16, 3, 1), ("stem", 5, 3, 64, 64, 8, 3, 1)]


@pytest.mark.timeout(300)
@pytest.mark.parametrize("kind,n,cin,cout,h,w,ks,stride", STAT_CASES)
def test_batchnorm_statistics_exact(kind, n, cin, cout, h, w, ks, stride, monkeypatch):
    from draco_b200.ops.conv import BnStatRequest, conv3x3_halo, conv_stem_fprop, convg_tcgen05
    g = _gen(n + cin + cout + h)
    K = ks * ks * cin
    x, wt = _iop((n, cin, h, w), K, g, target=16), _iop((cout, cin, ks, ks), K, g, target=16)
    bias = ((torch.arange(cout, device=DEV) % 7) - 3).float()              # small integer channel means
    ref_y = X.bf16_rn(X.conv_ref(x, wt, stride, bias))
    rm0 = torch.randint(-4, 5, (cout,), generator=g).float().to(DEV) * 0.25
    rv0 = torch.rand(cout, generator=g).to(DEV) + 0.5

    def launch():
        req = BnStatRequest(1e-5, 0.1, rm0.clone(), rv0.clone())
        if kind == "tap":
            y = convg_tcgen05(X.cl(x), X.wt(wt), (h, w), stride, False, bias, bn_stats=req)
        elif kind == "halo":
            y = conv3x3_halo(X.cl(x), X.wt(wt), False, bias, bn_stats=req)
        else:
            y = conv_stem_fprop(X.cl(x), X.wt(wt), bias, bn_stats=req)
        X.assert_equal(y, ref_y, f"{kind} output")
        _check_stats(req, ref_y, rm0, rv0, kind)
        return req

    req = launch()
    variants = [(e, c) for e, c in _variants(n, cin, cout, h, w, ks, stride, 0) if e == "tma"] if kind == "tap" else []
    for epi, cfg in variants:                                              # every tile width / cluster shape: same statistics
        _set_variant(monkeypatch, epi, cfg)
        r2 = launch()
        X.assert_equal(r2.mean, req.mean, f"mean [{cfg}]")
        X.assert_equal(r2.invstd, req.invstd, f"invstd [{cfg}]")
    from draco_b200.ops.norm import _lib as bn_lib
    if bn_lib().drc_bn_supported(cout):
        mean, invstd, rm, rv = _standalone_stats(ref_y, 1e-5, 0.1, rm0, rv0)
        X.assert_equal(mean, req.mean, "standalone vs epilogue: mean")
        X.assert_equal(invstd, req.invstd, "standalone vs epilogue: invstd")
        X.assert_equal(rm, req.running_mean, "standalone vs epilogue: running_mean")
        X.assert_equal(rv, req.running_var, "standalone vs epilogue: running_var")


@pytest.mark.parametrize("path", ["epilogue", "standalone"])
def test_batchnorm_invstd_bound_at_large_mean_to_std_ratio(path):
    """Real-valued channels with |mean| / std in {0, 1, 8, 64}.  var = E[y^2] - mean^2 in fp32 cancels: with fp32 sums of M terms
    (relative error <= gamma = M * 2^-23 each, any order) and the finalisation's own roundings,

        |var_k - var| <= (3 gamma + 10 * 2^-24) * E[y^2]  =: delta * var,   delta = (3 gamma + 10 * 2^-24) (1 + (mean/std)^2),

    so |invstd_k / invstd - 1| <= delta / (2 (1 - delta)) + 2^-22 (rsqrtf).  M = 256 keeps delta < 0.4 at ratio 64; the contract
    is this bound, i.e. a relative invstd error that grows with (mean / std)^2."""
    from draco_b200.ops.conv import BnStatRequest, convg_tcgen05
    n, h, w, c = 4, 8, 8, 64
    g = _gen(31)
    ratio = torch.tensor([0.0, 1.0, 8.0, 64.0]).repeat(c // 4)
    sign = 1 - 2 * (torch.arange(c) % 3 == 0).float()
    std = 1.0
    x = torch.randn(n, c, h, w, generator=g).to(torch.bfloat16).to(DEV)
    mean_c = (ratio * sign * std).to(DEV)
    eye = torch.eye(c, device=DEV).view(c, c, 1, 1)                      # identity 1x1 conv: y = bf16(x + mean_c)
    req = BnStatRequest(1e-5, 0.1)
    y = convg_tcgen05(X.cl(x), X.wt(eye), (h, w), 1, False, mean_c.float(), bn_stats=req)
    if path == "standalone":
        mean, invstd, _, _ = _standalone_stats(y, 1e-5, 0.1, torch.zeros(c, device=DEV), torch.ones(c, device=DEV))
    else:
        mean, invstd = req.mean, req.invstd
    yd = y.double()
    M = n * h * w
    m64 = yd.mean((0, 2, 3))
    var64 = yd.var((0, 2, 3), unbiased=False)
    e2 = (yd * yd).mean((0, 2, 3))
    inv64 = 1.0 / (var64 + 1e-5).sqrt()
    delta = (3 * M * 2.0 ** -23 + 10 * 2.0 ** -24) * e2 / (var64 + 1e-5)
    assert float(delta.max()) < 0.5
    bound = delta / (2 * (1 - delta)) + 2.0 ** -22
    err = (invstd.double() - inv64).abs() / inv64
    worst = int((err / bound).argmax())
    assert bool((err <= bound).all()), (f"channel {worst}: |mean|/std {float(ratio[worst])}, invstd rel. error {float(err[worst]):.3e} "
                                        f"> bound {float(bound[worst]):.3e}")
    assert bool(((mean.double() - m64).abs() <= M * 2.0 ** -23 * yd.abs().mean((0, 2, 3)) + 2.0 ** -23 * m64.abs()).all())


# ------------------------------------------------------------------------------------------------------------------------------
# BatchNorm-backward sums in the dgrad epilogue (BnBwdLink): dbeta = sum dz, dgamma = sum dz * xhat
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.timeout(300)
@pytest.mark.parametrize("kind,n,c,cout,h,w", [("tap", 5, 128, 192, 4, 8), ("tap", 3, 320, 64, 16, 4), ("halo", 3, 64, 64, 16, 64)])
@pytest.mark.parametrize("mask", ["y>0", "-y>0", "none"])
@pytest.mark.parametrize("with_res", [False, True])
def test_bn_backward_sums_in_dgrad_epilogue_exact(kind, n, c, cout, h, w, mask, with_res):
    """Integer dy / weights / x, integer BatchNorm mean and power-of-two invstd: xhat = (x - mean) * invstd is exact in fp32, so
    dz, sum(dz) and sum(dz * xhat) are all exact; the masked output and the four sums must match bit for bit."""
    from draco_b200.ops.conv import BnBwdLink, conv3x3_halo, convg_tcgen05
    g = _gen(n + c + h + len(mask) + with_res)
    wt = _iop((cout, c, 3, 3), 9 * cout, g, target=64)
    dy = _iop((n, cout, h, w), 9 * cout, g, target=64)
    xbn = torch.randint(-8, 9, (n, c, h, w), generator=g).float().to(DEV)           # input of the BatchNorm
    ybn = torch.randint(-2, 3, (n, c, h, w), generator=g).float().to(DEV)           # its output (this conv's input): zeros included
    mean = (torch.randint(-3, 4, (c,), generator=g)).float().to(DEV)
    invstd = torch.full((c,), 0.25, device=DEV)
    res = (torch.randint(-20, 21, (n, c, h, w), generator=g)).float().to(DEV) if with_res else None
    mtensor = ybn if mask == "y>0" else -ybn
    link = BnBwdLink(X.cl(xbn), mean, invstd, mask != "none")
    args = (X.cl(dy), X.wt(wt))
    rb = X.cl(res) if with_res else None
    if kind == "halo":
        dz = conv3x3_halo(*args, True, None, None, rb, (link, X.cl(mtensor)))
    else:
        dz = convg_tcgen05(*args, (h, w), 1, True, None, None, rb, (link, X.cl(mtensor)))
    dx64 = X.dgrad_ref(dy, wt, (h, w), 1) + (res.double() if with_res else 0)
    keep = (mtensor > 0) if mask != "none" else torch.ones_like(mtensor, dtype=torch.bool)
    ref_dz = X.bf16_rn(dx64 * keep)
    X.assert_equal(dz, ref_dz, "dz")
    assert link.dz is dz
    dzd = ref_dz.double()
    xhat = (xbn.double() - mean.double().view(1, -1, 1, 1)) * 0.25
    dbeta = dzd.sum((0, 2, 3))
    dgamma = (dzd * xhat).sum((0, 2, 3))
    X.assert_exact_domain(dzd.abs().sum((0, 2, 3)), 4 * (dzd * xhat).abs().sum((0, 2, 3)))
    X.assert_equal(link.dbeta, dbeta.float(), "dbeta = sum dz")
    X.assert_equal(link.dgamma, dgamma.float(), "dgamma = sum dz * xhat")
    inv_m = torch.tensor(1.0 / (n * h * w), dtype=torch.float32).double()
    X.assert_equal(link.sums[:c], (dbeta * inv_m).float(), "sums[0] = sum dz / M")
    X.assert_equal(link.sums[c:], (dgamma * inv_m).float(), "sums[1] = sum dz * xhat / M")


@pytest.mark.parametrize("kind", ["tap", "halo"])
def test_bn_backward_dgamma_randn_component_bound(kind):
    """Real-valued: dgamma = sum over M pixels of dz * xhat, xhat = (x - mean) * invstd rounded twice in fp32, fma-accumulated:
    |dgamma - ref64| <= (M + 3) * 2^-23 * sum |dz| |xhat|."""
    from draco_b200.ops.conv import BnBwdLink, conv3x3_halo, convg_tcgen05
    n, c, h, w = 3, 64, 16, 64
    g = _gen(41)
    wt = (torch.randn(64, c, 3, 3, generator=g) * 0.05).to(torch.bfloat16).to(DEV)
    dy = torch.randn(n, 64, h, w, generator=g).to(torch.bfloat16).to(DEV)
    xbn = (torch.randn(n, c, h, w, generator=g) * 2 + 0.5).to(torch.bfloat16).to(DEV)
    ybn = torch.randn(n, c, h, w, generator=g).to(torch.bfloat16).to(DEV)
    mean = xbn.float().mean((0, 2, 3))
    invstd = xbn.float().var((0, 2, 3), unbiased=False).add(1e-5).rsqrt()
    link = BnBwdLink(X.cl(xbn), mean, invstd, True)
    if kind == "halo":
        dz = conv3x3_halo(X.cl(dy), X.wt(wt), True, None, None, None, (link, X.cl(ybn)))
    else:
        dz = convg_tcgen05(X.cl(dy), X.wt(wt), (h, w), 1, True, None, None, None, (link, X.cl(ybn)))
    dzd = dz.double()
    xhat = (xbn.double() - mean.double().view(1, -1, 1, 1)) * invstd.double().view(1, -1, 1, 1)
    M = n * h * w
    assert bool(((link.dbeta.double() - dzd.sum((0, 2, 3))).abs() <= (M + 1) * 2.0 ** -23 * dzd.abs().sum((0, 2, 3))).all())
    X.assert_bound(link.dgamma, (dzd * xhat).sum((0, 2, 3)), (dzd * xhat).abs().sum((0, 2, 3)), M + 2, "dgamma", rel=0.0)


# ------------------------------------------------------------------------------------------------------------------------------
# head kernels: fused cross-entropy (csrc/cuda/loss_fused.cu), Prec@k ties, global average pool (csrc/cuda/pool_head.cu)
# ------------------------------------------------------------------------------------------------------------------------------
def _ce_run(logits, labels):
    from draco_b200.ops.loss import cross_entropy_with_metrics, fused_enabled
    assert fused_enabled(logits)
    metrics = torch.zeros(3, device=DEV)
    lg = logits.clone().requires_grad_(True)
    loss = cross_entropy_with_metrics(lg, labels, metrics, 1.0)
    loss.backward()
    return loss.detach(), lg.grad, metrics


def _prec_ref(logits, labels, k):
    """Documented rule: a row counts for Prec@k when fewer than k logits are strictly greater than the label's."""
    z = logits.double()
    zl = z.gather(1, labels.view(-1, 1))
    return int(((z > zl).sum(1) < k).sum())


def _metric_f32(count, B):
    t = torch.tensor(100.0, dtype=torch.float32) * torch.tensor(1.0 / B, dtype=torch.float32).float()
    return (torch.tensor(float(count), dtype=torch.float32) * t).item()


@pytest.mark.parametrize("B,C,dtype,scale", [(300, 32, torch.bfloat16, 8.0), (300, 33, torch.bfloat16, 8.0), (128, 10, torch.float32, 4.0),
                                             (300, 100, torch.float32, 8.0), (77, 100, torch.bfloat16, 80.0), (129, 33, torch.float32, 80.0),
                                             (5, 1000, torch.bfloat16, 3.0)])
def test_fused_cross_entropy_against_fp64(B, C, dtype, scale):
    """Loss, gradient and Prec@1/5 of the fused kernel against an fp64 log-softmax.  Bounds: __expf is within 2 + 1.173 |x| ulp,
    i.e. 2^-15.4 relative for x in [-160, 0]; the sum of C <= 1000 terms adds C 2^-24 <= 2^-14, so e / sum(e) is within
    2^-13.2 p -- taken as 2^-12 p -- and a row's loss within 2^-12 + 2^-22 (|lse| + |z_label|); the mean over B rows adds
    (B + 1) 2^-23 of the absolute row sum.  The gradient (p - onehot) / B gets 2^-12 p / B + its roundings (2^-8 relative in bf16,
    2^-21 in fp32: subtraction, 1/B and product) + 2^-100 absolute (exp underflow below the fp32 range)."""
    g = _gen(B + C)
    logits = ((torch.rand(B, C, generator=g) * 2 - 1) * scale).to(dtype).to(DEV)    # scale 80: logits of +-80
    labels = torch.randint(0, C, (B,), generator=g).to(DEV)
    loss, grad, metrics = _ce_run(logits, labels)
    z = logits.double()
    lse = torch.logsumexp(z, 1)
    zl = z.gather(1, labels.view(-1, 1)).squeeze(1)
    row = lse - zl
    tol = float((2.0 ** -12 + 2.0 ** -22 * (lse.abs() + zl.abs())).mean() + (B + 1) * 2.0 ** -23 * row.abs().mean())
    assert abs(float(loss) - float(row.mean())) <= tol, (float(loss), float(row.mean()), tol)
    p = torch.softmax(z, 1)
    g64 = (p - torch.nn.functional.one_hot(labels, C).double()) / B
    rel = 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -21
    bound = 2.0 ** -12 * p / B + rel * g64.abs() + 2.0 ** -100
    err = (grad.double() - g64).abs()
    assert grad.dtype == dtype and bool((err <= bound).all()), f"worst at {divmod(int((err / bound).argmax()), C)}"
    assert metrics[0].item() == loss.item()
    assert metrics[1].item() == _metric_f32(_prec_ref(logits, labels, 1), B)
    assert metrics[2].item() == _metric_f32(_prec_ref(logits, labels, 5), B)


@pytest.mark.parametrize("B,C,dtype", [(300, 10, torch.bfloat16), (300, 10, torch.float32), (300, 33, torch.bfloat16),
                                       (130, 100, torch.float32), (64, 32, torch.bfloat16)])
def test_prec_at_k_ties_with_integer_logits(B, C, dtype):
    """Integer logits in {0, 1, 2, 3}: most rows have ties with the label's logit; ties count for the label."""
    g = _gen(B * C)
    logits = torch.randint(0, 4, (B, C), generator=g).to(dtype).to(DEV)
    labels = torch.randint(0, C, (B,), generator=g).to(DEV)
    p1, p5 = _prec_ref(logits, labels, 1), _prec_ref(logits, labels, 5)
    ties = int((logits.double() == logits.double().gather(1, labels.view(-1, 1))).sum()) - B
    assert ties > B                                                       # the case is really tie-heavy
    _, _, metrics = _ce_run(logits, labels)
    assert metrics[1].item() == _metric_f32(p1, B)
    assert metrics[2].item() == _metric_f32(p5, B)


@pytest.mark.parametrize("n,c,h,w", [(3, 64, 2, 8), (5, 128, 8, 2), (2, 512, 4, 1), (4, 256, 16, 4), (2, 64, 1, 32)])
def test_global_avg_pool_exact_on_non_square_inputs(n, c, h, w):
    """Even integers |x| <= 300 (exact in bf16) over a power-of-two H * W: the fp32 sum and the 1/HW scale are exact, so the bf16
    mean must equal the exact mean rounded once; the backward dy / HW is exact."""
    from draco_b200.ops.pool import backend_counters, global_avg_pool
    g = _gen(n * c + h)
    x = (torch.randint(-150, 151, (n, c, h, w), generator=g) * 2).float().to(DEV)
    xb = X.cl(x).requires_grad_(True)
    before = backend_counters["native"]
    y = global_avg_pool(xb)
    assert backend_counters["native"] == before + 1
    X.assert_equal(y, X.bf16_rn(x.double().mean((2, 3))), "pool forward")
    dy = torch.randn(n, c, generator=g).to(torch.bfloat16).to(DEV)
    y.backward(dy)
    X.assert_equal(xb.grad, (dy.double() / (h * w)).view(n, c, 1, 1).expand(n, c, h, w).to(torch.bfloat16), "pool backward")
