"""wgmma GEMM (csrc/cuda/gemm_wgmma.cu) and the Linear layer built on it, against fp32 PyTorch references."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def K():
    from draco_b200.ops import kernels
    return kernels


def _rel_err(a, b):
    return float((a.float() - b.float()).abs().max() / b.float().abs().max().clamp_min(1e-6))


SHAPES = [(128, 128, 64), (256, 192, 512), (300, 504, 784), (128, 800, 784), (77, 136, 72), (4096, 512, 4608),
          (1000, 16, 512), (64, 64, 8), (130, 264, 1032)]


@pytest.mark.parametrize("M,N,Kd", SHAPES)
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, False), (True, True)])
def test_gemm_all_operand_orders(K, M, N, Kd, a_mn, b_mn):
    dev = torch.device("cuda", 0)
    torch.manual_seed(M * 7 + N * 3 + Kd)
    if (a_mn and M % 8) or (b_mn and N % 8):
        pytest.skip("MN-major operand needs a 16-byte row pitch")
    A = torch.randn(M, Kd, device=dev).to(torch.bfloat16)
    B = torch.randn(N, Kd, device=dev).to(torch.bfloat16)
    ref = A.float() @ B.float().t()
    A_in = A.t().contiguous() if a_mn else A
    B_in = B.t().contiguous() if b_mn else B
    out = K.gemm_bf16(A_in, B_in, a_mn=a_mn, b_mn=b_mn, out_dtype=torch.float32)
    torch.cuda.synchronize()
    assert out.shape == (M, N)
    assert _rel_err(out, ref) < 2e-3, _rel_err(out, ref)
    out16 = K.gemm_bf16(A_in, B_in, a_mn=a_mn, b_mn=b_mn)
    assert _rel_err(out16, ref) < 1.5e-2


@pytest.mark.parametrize("block_n", [32, 64, 128, 256])
def test_gemm_block_n_variants_bias_relu_accumulate(K, block_n):
    dev = torch.device("cuda", 0)
    torch.manual_seed(block_n)
    M, N, Kd = 515, 328, 1000
    A = torch.randn(M, Kd, device=dev).to(torch.bfloat16)
    B = torch.randn(N, Kd, device=dev).to(torch.bfloat16)
    bias = torch.randn(N, device=dev)
    ref = torch.relu(A.float() @ B.float().t() + bias)
    out = K.gemm_bf16(A, B, out_dtype=torch.float32, bias=bias, relu=True, block_n=block_n)
    assert _rel_err(out, ref) < 2e-3
    out_b = K.gemm_bf16(A, B, bias=bias.to(torch.bfloat16), relu=True, block_n=block_n)
    assert _rel_err(out_b, ref) < 2e-2
    acc = torch.ones(M, N, device=dev)
    K.gemm_bf16(A, B, out=acc, accumulate=True, block_n=block_n)
    assert _rel_err(acc, A.float() @ B.float().t() + 1.0) < 2e-3


def test_gemm_odd_ldc_scalar_store_path(K):
    dev = torch.device("cuda", 0)
    A = torch.randn(200, 512, device=dev).to(torch.bfloat16)
    B = torch.randn(10, 512, device=dev).to(torch.bfloat16)       # the CIFAR classifier: N = 10
    ref = A.float() @ B.float().t()
    assert _rel_err(K.gemm_bf16(A, B, out_dtype=torch.float32), ref) < 2e-3
    assert _rel_err(K.gemm_bf16(A, B), ref) < 1.5e-2


def test_gemm_is_deterministic(K):
    dev = torch.device("cuda", 0)
    A = torch.randn(1024, 2048, device=dev).to(torch.bfloat16)
    B = torch.randn(768, 2048, device=dev).to(torch.bfloat16)
    o1 = K.gemm_bf16(A, B)
    o2 = K.gemm_bf16(A, B)
    assert torch.equal(o1, o2)


@pytest.mark.parametrize("batch,fin,fout", [(128, 512, 512), (128, 784, 800), (128, 512, 10), (96, 800, 500)])
def test_linear_layer_forward_backward(batch, fin, fout):
    from draco_b200.ops.linear import Linear, backend_counters
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    lin = Linear(fin, fout).to(dev).to(torch.bfloat16)
    x = torch.randn(batch, fin, device=dev).to(torch.bfloat16).requires_grad_(True)
    before = backend_counters["tcgen05"]
    y = lin(x)
    gy = torch.randn_like(y)
    y.backward(gy)
    assert backend_counters["tcgen05"] > before, "the tensor-core path did not run"
    w32, b32 = lin.weight.detach().float().requires_grad_(True), lin.bias.detach().float().requires_grad_(True)
    x32 = x.detach().float().requires_grad_(True)
    y32 = F.linear(x32, w32, b32)
    y32.backward(gy.float())
    assert _rel_err(y, y32) < 1.5e-2
    assert _rel_err(x.grad, x32.grad) < 2e-2
    assert _rel_err(lin.weight.grad, w32.grad) < 2e-2
    assert _rel_err(lin.bias.grad, b32.grad) < 2e-2


@pytest.mark.parametrize("n,cin,cout,hw", [(32, 64, 256, 16), (16, 256, 64, 8), (8, 512, 2048, 4), (128, 64, 64, 32)])
def test_pointwise_conv_on_tcgen05(n, cin, cout, hw):
    from draco_b200.ops.conv import Conv2d, backend_counters
    dev = torch.device("cuda", 0)
    torch.manual_seed(cin + cout)
    conv = Conv2d(cin, cout, kernel_size=1, bias=False).to(dev).to(torch.bfloat16).to(memory_format=torch.channels_last)
    x = torch.randn(n, cin, hw, hw, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    before = backend_counters["tcgen05"]
    y = conv(x)
    assert backend_counters["tcgen05"] == before + 1
    assert y.shape == (n, cout, hw, hw) and y.is_contiguous(memory_format=torch.channels_last)
    gy = torch.randn_like(y)
    y.backward(gy)
    x32 = x.detach().float().requires_grad_(True)
    w32 = conv.weight.detach().float().requires_grad_(True)
    y32 = F.conv2d(x32, w32)
    y32.backward(gy.float())
    assert _rel_err(y, y32) < 1.5e-2
    assert _rel_err(x.grad, x32.grad) < 2e-2
    assert _rel_err(conv.weight.grad, w32.grad) < 2e-2
    # geometries no native kernel serves (5x5 here) take the library path
    c5 = Conv2d(cin, cout, kernel_size=5, padding=2, bias=False).to(dev).to(torch.bfloat16)
    b2 = backend_counters["cudnn"]
    c5(x.detach())
    assert backend_counters["cudnn"] == b2 + 1


def _cl(t):
    return t.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)


def _wt(cout, cin, ks, dev, scale=0.05):
    w = (torch.randn(cout, cin, ks, ks, device=dev) * scale).to(torch.bfloat16)
    return w.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)               # [Cout, ks, ks, Cin] storage (arena layout)


def _bn_ref(y):
    yf = y.float()
    mean = yf.mean((0, 2, 3))
    var = yf.var((0, 2, 3), unbiased=False)
    return mean, (var + 1e-5).rsqrt(), yf.var((0, 2, 3), unbiased=True)


TAP_SHAPES = [(128, 64, 128, 32, 3, 2), (128, 128, 256, 16, 3, 2), (128, 256, 512, 8, 3, 2), (128, 64, 128, 32, 1, 2),
              (64, 128, 256, 16, 1, 2), (5, 256, 512, 8, 1, 2), (8, 64, 64, 32, 3, 1), (16, 128, 128, 16, 3, 1), (6, 64, 128, 16, 1, 1),
              (128, 128, 128, 16, 3, 1), (128, 256, 256, 8, 3, 1), (128, 512, 512, 4, 3, 1), (7, 512, 64, 2, 3, 1), (3, 128, 192, 4, 3, 1),
              (32, 512, 512, 2, 3, 1),
              # ImageNet-ResNet geometries: image sizes that are not powers of two tile exactly as well (8 x 8 x 2, 4 x 4 x 8, ...)
              (6, 64, 64, 56, 3, 1), (6, 128, 128, 28, 3, 1), (9, 256, 256, 14, 3, 1), (20, 512, 512, 7, 3, 1), (6, 64, 128, 56, 3, 2),
              (5, 256, 512, 14, 1, 2), (3, 64, 256, 56, 1, 1)]


@pytest.mark.timeout(300)
@pytest.mark.parametrize("epi", ["tma", "direct"])
@pytest.mark.parametrize("n,cin,cout,hw,ks,stride", TAP_SHAPES)
def test_convg_tap_table_kernels(n, cin, cout, hw, ks, stride, epi, monkeypatch):
    """Tap-table wgmma implicit GEMM (csrc/cuda/conv_tap_wgmma.cu): fprop / dgrad / split-K wgrad for 3x3 and 1x1, stride 1 and
    2, with the staged TMA-store epilogue and with the direct-store epilogue, against fp32 references."""
    from draco_b200.ops.conv import convg_tcgen05, convg_wgrad_tcgen05
    monkeypatch.setenv("DRACO_CONV_EPI", epi)
    dev = torch.device("cuda", 0)
    torch.manual_seed(n + cin + cout + hw + ks + stride)
    pad = ks // 2
    x = _cl(torch.randn(n, cin, hw, hw, device=dev))
    w = _wt(cout, cin, ks, dev)
    b = torch.randn(cout, device=dev)
    y = convg_tcgen05(x, w, (hw, hw), stride, False, b)
    ref = F.conv2d(x.float(), w.float(), b, stride=stride, padding=pad)
    assert y.shape == ref.shape and y.is_contiguous(memory_format=torch.channels_last) and _rel_err(y, ref) < 1.5e-2, _rel_err(y, ref)
    dy = _cl(torch.randn_like(ref))
    dx = convg_tcgen05(dy, w, (hw, hw), stride, True)
    dref = torch.nn.grad.conv2d_input(x.shape, w.float(), dy.float(), stride=stride, padding=pad)
    assert dx.shape == dref.shape and _rel_err(dx, dref) < 1.5e-2, _rel_err(dx, dref)
    if epi == "tma":
        dw = convg_wgrad_tcgen05(dy, x, ks, stride)
        wref = torch.nn.grad.conv2d_weight(x.float(), (cout, cin, ks, ks), dy.float(), stride=stride, padding=pad)
        assert dw.shape == wref.shape and _rel_err(dw, wref) < 1.5e-2, _rel_err(dw, wref)
        assert torch.equal(convg_wgrad_tcgen05(dy, x, ks, stride), dw)      # deterministic split-K
    assert torch.equal(convg_tcgen05(x, w, (hw, hw), stride, False, b), y)  # deterministic


@pytest.mark.timeout(300)
@pytest.mark.parametrize("n,cin,cout,hw,ks,stride", [(128, 64, 64, 32, 3, 1), (16, 128, 128, 16, 3, 1), (128, 64, 128, 32, 3, 2),
                                                     (5, 256, 512, 8, 3, 2), (7, 512, 64, 2, 3, 1), (6, 64, 64, 56, 3, 1)])
def test_conv_dgrad_epilogue_adds_fork_gradient(n, cin, cout, hw, ks, stride):
    """dgrad with a residual tensor added in the epilogue (halo kernel, dense tap kernel, one-launch stride-2 tap kernel): equals
    the plain dgrad plus the tensor in fp32, rounded once; and through autograd a forked input (residual block) gets the same
    gradient as conv + identity shortcut in fp32."""
    from draco_b200.ops.conv import Conv2d, conv3x3_halo, convg_tcgen05, halo_supported
    dev = torch.device("cuda", 0)
    torch.manual_seed(n + cin + hw + stride)
    w = _wt(cout, cin, ks, dev)
    dy = _cl(torch.randn(n, cout, hw // stride, hw // stride, device=dev))
    r = _cl(torch.randn(n, cin, hw, hw, device=dev))
    ref = torch.nn.grad.conv2d_input((n, cin, hw, hw), w.float(), dy.float(), stride=stride, padding=ks // 2) + r.float()
    dx = convg_tcgen05(dy, w, (hw, hw), stride, True, None, None, r)
    assert _rel_err(dx, ref) < 1.5e-2, _rel_err(dx, ref)
    assert torch.equal(dx, convg_tcgen05(dy, w, (hw, hw), stride, True, None, None, r))
    if stride == 1 and halo_supported(hw, hw, cin, cout):
        dxh = conv3x3_halo(dy, w, True, None, None, r)
        assert _rel_err(dxh, ref) < 1.5e-2, _rel_err(dxh, ref)
    # autograd: y = conv(x) ; z = y.sum-like + fork
    conv = Conv2d(cin, cout, kernel_size=ks, stride=stride, padding=ks // 2, bias=False).to(dev).to(torch.bfloat16)
    conv.weight.data = w.clone()
    x = _cl(torch.randn(n, cin, hw, hw, device=dev)).requires_grad_(True)
    y, xf = conv(x, fork=True)
    gz = _cl(torch.randn_like(y))
    (y.float() * gz.float()).sum().add((xf.float() * r.float()).sum()).backward()
    x32 = x.detach().float().requires_grad_(True)
    y32 = F.conv2d(x32, w.float(), stride=stride, padding=ks // 2)
    ((y32 * gz.float()).sum() + (x32 * r.float()).sum()).backward()
    assert _rel_err(x.grad, x32.grad) < 2e-2, _rel_err(x.grad, x32.grad)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("cfg", ["2,1,128", "1,2,128", "2,2,128", "4,2,128", "2,4,64", "8,1,64", "1,8,64", "4,1,128", "1,4,64",
                                 "2,1,64", "1,2,64", "2,2,64", "4,2,64"])
@pytest.mark.parametrize("n,cin,cout,hw,ks,stride", [(128, 256, 256, 8, 3, 1), (128, 512, 512, 4, 3, 1), (128, 128, 256, 16, 3, 2),
                                                     (24, 64, 512, 14, 1, 1)])
def test_convg_cluster_multicast_shapes(n, cin, cout, hw, ks, stride, cfg, monkeypatch):
    """Cluster variants of the tap convolution.  "cm,cn,bn": every CTA loads 1/cn of the activation tile and 1/cm of the
    weight tile and TMA-multicasts them to its cluster row / column.  Each forced shape must reproduce the one-CTA-per-tile kernel
    (same k order per output element) for fprop (with fused BatchNorm statistics), dense dgrad and the one-launch stride-2 dgrad."""
    from draco_b200.ops.conv import BnStatRequest, convg_plan, convg_tcgen05
    dev = torch.device("cuda", 0)
    torch.manual_seed(n + cin + hw)
    x = _cl(torch.randn(n, cin, hw, hw, device=dev))
    w = _wt(cout, cin, ks, dev)
    dy = _cl(torch.randn(n, cout, hw // stride, hw // stride, device=dev))
    monkeypatch.setenv("DRACO_CONV_CLUSTER", "1,1")
    ra = BnStatRequest(1e-5, 0.1)
    y0 = convg_tcgen05(x, w, (hw, hw), stride, False, None, bn_stats=ra)
    dx0 = convg_tcgen05(dy, w, (hw, hw), stride, True)
    ref = F.conv2d(x.float(), w.float(), None, stride=stride, padding=ks // 2)
    assert _rel_err(y0, ref) < 1.5e-2
    monkeypatch.setenv("DRACO_CONV_CLUSTER", cfg)
    def forced(dgrad):
        plan = convg_plan(n, hw, hw, cin, cout, ks, stride, dgrad)
        cm, cn, bn = (int(v) for v in cfg.split(","))
        return plan[:3] == [bn, cm, cn] and plan[4] == 1

    ran = 0
    if forced(0):
        rb = BnStatRequest(1e-5, 0.1)
        y1 = convg_tcgen05(x, w, (hw, hw), stride, False, None, bn_stats=rb)
        assert torch.equal(y0, y1)
        assert _rel_err(rb.mean, ra.mean) < 1e-5 and _rel_err(rb.invstd, ra.invstd) < 1e-5
        assert torch.equal(convg_tcgen05(x, w, (hw, hw), stride, False, None), y1)
        ran += 1
    if forced(1):
        assert torch.equal(convg_tcgen05(dy, w, (hw, hw), stride, True), dx0)
        ran += 1
    if not ran:
        pytest.skip("cluster shape not realisable for this layer")


@pytest.mark.timeout(300)
@pytest.mark.parametrize("n,cin,cout,hw,ks,stride", [(128, 64, 128, 32, 3, 2), (128, 128, 128, 16, 3, 1), (128, 256, 256, 8, 3, 1),
                                                     (128, 512, 512, 4, 3, 1), (9, 64, 128, 32, 1, 2), (5, 256, 512, 8, 3, 2),
                                                     (3, 128, 192, 4, 3, 1), (128, 128, 256, 16, 1, 2)])
def test_conv_epilogue_batchnorm_statistics(n, cin, cout, hw, ks, stride):
    """The convolution epilogue's fused BatchNorm statistics (csrc/cuda/conv_epilogue.cuh): mean / invstd of the bf16 output and the
    running-statistics momentum update, vs torch on the kernel's own output; deterministic; with a conv bias and partial tiles."""
    from draco_b200.ops.conv import BnStatRequest, convg_tcgen05
    dev = torch.device("cuda", 0)
    torch.manual_seed(n + cin + hw)
    x = _cl(torch.randn(n, cin, hw, hw, device=dev))
    w = _wt(cout, cin, ks, dev)
    b = torch.randn(cout, device=dev)
    rm, rv = torch.zeros(cout, device=dev), torch.ones(cout, device=dev)
    req = BnStatRequest(1e-5, 0.1, rm, rv)
    y = convg_tcgen05(x, w, (hw, hw), stride, False, b, bn_stats=req)
    mean, invstd, unbiased = _bn_ref(y)
    assert _rel_err(req.mean, mean) < 1e-4 and _rel_err(req.invstd, invstd) < 1e-3, (_rel_err(req.mean, mean), _rel_err(req.invstd, invstd))
    assert _rel_err(rm, 0.1 * mean) < 1e-4 and _rel_err(rv, 0.9 + 0.1 * unbiased) < 1e-3
    req2 = BnStatRequest(1e-5, 0.1)
    y2 = convg_tcgen05(x, w, (hw, hw), stride, False, b, bn_stats=req2)
    assert torch.equal(y, y2) and torch.equal(req.mean, req2.mean) and torch.equal(req.invstd, req2.invstd)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("n,hw", [(4, 32), (128, 32), (3, 16), (16, 64)])
def test_conv3x3_halo_reuse_kernels(n, hw):
    """Halo loaded once per tile as three column-shifted boxes, tap (r, s) = box s from row r on (64 -> 64 channels), resident weights, staged
    TMA-store epilogue with fused BatchNorm statistics (csrc/cuda/conv_halo_wgmma.cu)."""
    from draco_b200.ops.conv import BnStatRequest, conv3x3_halo
    dev = torch.device("cuda", 0)
    torch.manual_seed(n + hw)
    x = _cl(torch.randn(n, 64, hw, hw, device=dev))
    w = _wt(64, 64, 3, dev)
    b = torch.randn(64, device=dev)
    req = BnStatRequest(1e-5, 0.1)
    y = conv3x3_halo(x, w, False, b, bn_stats=req)
    ref = F.conv2d(x.float(), w.float(), b, padding=1)
    assert _rel_err(y, ref) < 1.5e-2, _rel_err(y, ref)
    mean, invstd, _ = _bn_ref(y)
    assert _rel_err(req.mean, mean) < 1e-4 and _rel_err(req.invstd, invstd) < 1e-3
    dy = _cl(torch.randn(n, 64, hw, hw, device=dev))
    dx = conv3x3_halo(dy, w, True)
    dref = torch.nn.grad.conv2d_input(x.shape, w.float(), dy.float(), padding=1)
    assert _rel_err(dx, dref) < 1.5e-2, _rel_err(dx, dref)
    assert torch.equal(conv3x3_halo(x, w, False, b), y)
    # weight gradient: all nine taps from one resident halo patch (tap pairs stacked in M, MN-major views of the patch)
    from draco_b200.ops.conv import conv3x3_halo_wgrad
    dw = conv3x3_halo_wgrad(dy, x)
    wref = torch.nn.grad.conv2d_weight(x.float(), (64, 64, 3, 3), dy.float(), padding=1)
    assert dw.shape == wref.shape and _rel_err(dw, wref) < 1.5e-2, _rel_err(dw, wref)
    assert torch.equal(conv3x3_halo_wgrad(dy, x), dw)


@pytest.mark.timeout(300)
def test_conv_layer_autograd_paths_are_native():
    """ops.conv.Conv2d: every ResNet / VGG geometry (3x3 and 1x1, stride 1 and 2, stem) is served by this repository's kernels --
    the library counter must not move -- and matches fp32 autograd."""
    from draco_b200.ops.conv import Conv2d, backend_counters
    dev = torch.device("cuda", 0)
    torch.manual_seed(9)
    for cin, cout, ks, stride, hw in [(64, 64, 3, 1, 32), (64, 128, 3, 2, 32), (64, 128, 1, 2, 32), (128, 128, 3, 1, 16), (512, 512, 3, 1, 4),
                                      (3, 64, 3, 1, 32), (256, 64, 1, 1, 8)]:
        conv = Conv2d(cin, cout, ks, stride=stride, padding=ks // 2, bias=False).to(dev).to(torch.bfloat16).to(memory_format=torch.channels_last)
        x = _cl(torch.randn(16, cin, hw, hw, device=dev)).requires_grad_(cin != 3)
        lib_before = backend_counters["cudnn"]
        y = conv(x)
        gy = torch.randn_like(y)
        y.backward(gy)
        assert backend_counters["cudnn"] == lib_before, (cin, cout, ks, stride)
        x32, w32 = x.detach().float().requires_grad_(cin != 3), conv.weight.detach().float().requires_grad_(True)
        y32 = F.conv2d(x32, w32, stride=stride, padding=ks // 2)
        y32.backward(gy.float())
        assert _rel_err(y, y32) < 1.5e-2 and _rel_err(conv.weight.grad, w32.grad) < 2e-2, (cin, cout, ks, stride)
        if cin != 3:
            assert _rel_err(x.grad, x32.grad) < 2e-2


@pytest.mark.timeout(300)
@pytest.mark.parametrize("n,hw", [(128, 32), (5, 32), (16, 16), (3, 64), (2, 8 * 4)])
def test_conv_stem_native_kernels(n, hw):
    from draco_b200.ops.conv import BnStatRequest, conv_stem_fprop, conv_stem_wgrad
    dev = torch.device("cuda", 0)
    torch.manual_seed(n + hw)
    x = _cl(torch.randn(n, 3, hw, hw, device=dev))
    w = _wt(64, 3, 3, dev, 0.2)
    b = torch.randn(64, device=dev)
    req = BnStatRequest(1e-5, 0.1)
    y = conv_stem_fprop(x, w, b, bn_stats=req)
    ref = F.conv2d(x.float(), w.float(), b, padding=1)
    assert y.shape == ref.shape and y.is_contiguous(memory_format=torch.channels_last) and _rel_err(y, ref) < 1e-2
    mean, invstd, _ = _bn_ref(y)
    assert _rel_err(req.mean, mean) < 1e-4 and _rel_err(req.invstd, invstd) < 1e-3
    assert torch.equal(conv_stem_fprop(x, w, b), y)
    dy = _cl(torch.randn(n, 64, hw, hw, device=dev))
    dw = conv_stem_wgrad(dy, x)
    wref = torch.nn.grad.conv2d_weight(x.float(), (64, 3, 3, 3), dy.float(), padding=1)
    assert dw.shape == wref.shape and _rel_err(dw, wref) < 1e-2, _rel_err(dw, wref)
    assert torch.equal(conv_stem_wgrad(dy, x), dw)


@pytest.mark.timeout(300)
def test_resnet_block_conv_bn_fusion_matches_unfused(monkeypatch):
    """A BasicBlock forward / backward with the statistics taken from the convolution epilogues equals the same block with the
    standalone statistics kernel (same kernels otherwise) up to fp32 summation order, and uses no library convolution."""
    from draco_b200.models.resnet import BasicBlock
    from draco_b200.ops import norm
    from draco_b200.ops.conv import backend_counters
    dev = torch.device("cuda", 0)
    torch.manual_seed(1)
    blk = BasicBlock(64, 128, 2).to(dev)
    for m in blk.modules():
        if isinstance(m, torch.nn.Conv2d):
            m.to(torch.bfloat16)
    blk = blk.to(memory_format=torch.channels_last)
    x = _cl(torch.randn(32, 64, 32, 32, device=dev))
    outs = []
    for mode in ("conv", "kernel"):
        monkeypatch.setenv("DRACO_BN_STATS", mode)
        blk.zero_grad()
        for m in blk.modules():
            if isinstance(m, norm.FusedBatchNorm2d):
                m.reset_running_stats()
        lib_before, fused_before = backend_counters["cudnn"], norm.backend_counters.get("conv_stats", 0)
        xi = x.clone().requires_grad_(True)
        y = blk(xi)
        y.float().square().mean().backward()
        assert backend_counters["cudnn"] == lib_before
        assert (norm.backend_counters.get("conv_stats", 0) - fused_before) == (3 if mode == "conv" else 0)
        outs.append((y.detach().float(), xi.grad.float(), blk.conv1.weight.grad.float(), blk.bn2.running_var.clone()))
    for a, b in zip(*outs):
        assert _rel_err(a, b) < 2e-2, _rel_err(a, b)


@pytest.mark.timeout(300)
@pytest.mark.parametrize("planes,hw,n", [(64, 32, 32), (128, 16, 16), (256, 8, 128), (512, 4, 24)])
def test_batchnorm_backward_reduction_inside_the_dgrad_epilogue(planes, hw, n, monkeypatch):
    """Two stacked BasicBlocks: the BatchNorm backward reductions (sum dz, sum dz * xhat) of the layers whose output feeds a
    stride-1 convolution can ride on that convolution's dgrad epilogue (DRACO_BN_BWD_FUSE=1; halo and tap kernels, with the
    residual-fork gradient added first), so those BatchNorms only run their apply kernel.  Same result as the standalone reduce
    kernels up to summation order; deterministic; the counter proves the fused path ran.  (Opt-in.)"""
    from draco_b200.models.resnet import BasicBlock
    from draco_b200.ops import norm
    dev = torch.device("cuda", 0)
    torch.manual_seed(planes + hw)
    net = torch.nn.Sequential(BasicBlock(planes, planes, 1), BasicBlock(planes, planes, 1)).to(dev)
    for m in net.modules():
        if isinstance(m, torch.nn.Conv2d):
            m.to(torch.bfloat16)
    net = net.to(memory_format=torch.channels_last)
    bn0 = norm.FusedBatchNorm2d(planes).to(dev)
    x = _cl(torch.randn(n, planes, hw, hw, device=dev))
    gy = _cl(torch.randn(n, planes, hw, hw, device=dev))
    runs = {}
    for mode in ("1", "0", "1"):
        monkeypatch.setenv("DRACO_BN_BWD_FUSE", mode)
        net.zero_grad()
        bn0.zero_grad()
        before = norm.backend_counters.get("bwd_in_conv", 0)
        xi = x.clone().requires_grad_(True)
        y = net(bn0(xi, relu=True))            # bn0 -> block1.conv1 (fork) ; block1.bn1 -> conv2 ; block1 out -> block2.conv1 (fork) ; ...
        y.backward(gy)
        used = norm.backend_counters.get("bwd_in_conv", 0) - before
        assert used == (4 if mode == "1" else 0), used          # bn0, block1.bn1, block1.bn2 (block output), block2.bn1
        got = [xi.grad.float(), bn0.weight.grad.clone(), bn0.bias.grad.clone(), net[0].bn1.weight.grad.clone(),
               net[0].bn2.weight.grad.clone(), net[0].bn2.bias.grad.clone(), net[0].conv1.weight.grad.float(),
               net[1].bn1.bias.grad.clone()]
        if mode in runs:
            for a, b in zip(runs[mode], got):
                assert torch.equal(a, b)                          # deterministic
        runs[mode] = got
    for a, b in zip(runs["1"], runs["0"]):
        assert _rel_err(a, b) < 2e-2, _rel_err(a, b)
