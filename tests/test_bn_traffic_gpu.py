"""BatchNorm activation traffic (csrc/cuda/bn_fused.cu): the forward's 1-bit ReLU masks and the one-pass BatchNorm pair of a
downsampling block give exactly what the saved-output mask and two separate BatchNorm calls give."""
import pytest
import torch
import torch.nn.functional as F

import exact_ref as X

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)


def _cl(t):
    return t.contiguous(memory_format=torch.channels_last)


def _bits(t):
    """Bit pattern of a tensor (NaN compares equal to the same NaN)."""
    return t.contiguous().view({torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.int64: torch.int64}[t.dtype])


def _same(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _fwd_with_mask(x, res, scale, shift):
    """bn_apply_kernel with the given per-channel scale / shift (gamma = scale, invstd = 1, mean = 0): y and its ReLU bits."""
    from draco_b200.ops import norm
    lib = norm._lib()
    n, c, h, w = x.shape
    y = torch.empty_like(x)
    mask = torch.empty(n * h * w * c // 8, dtype=torch.uint8, device=DEV)
    ones, zeros = torch.ones(c, device=DEV), torch.zeros(c, device=DEV)
    from draco_b200 import _native as N
    N.check(lib.drc_bn_fwd(x.data_ptr(), None if res is None else res.data_ptr(), y.data_ptr(), mask.data_ptr(),
                           scale.data_ptr(), shift.data_ptr(), None, None, zeros.data_ptr(), ones.data_ptr(), None, None,
                           n * h * w, c, 1e-5, 0.1, 1, norm._sms(DEV), 1, torch.cuda.current_stream().cuda_stream), "bn_fwd")
    torch.cuda.synchronize()
    return y, mask


@pytest.mark.parametrize("shape", [(2, 8, 3, 5), (4, 64, 5, 5), (3, 512, 3, 3), (2, 2048, 1, 3), (3, 8, 5, 7), (7, 64, 9, 11)])
@pytest.mark.parametrize("with_res", [False, True])
def test_relu_bits_equal_stored_output_positive(shape, with_res):
    """Bit i of byte (row, cv) is bf16(y) > 0 for channel 8 cv + i, on +-0, values that round to bf16 zero, NaN, a residual
    that cancels the normalised value exactly, and ordinary values; M is not a multiple of the row groups."""
    torch.manual_seed(sum(shape))
    n, c, h, w = shape
    x = torch.randn(shape, device=DEV)
    k = x.numel()
    flat = x.view(-1)
    flat[0::7] = 0.0
    flat[1::7] = -0.0
    flat[2::7] = 2.0 ** -126                       # times 2^-20 below: positive in fp32, zero in bf16
    flat[3::7] = float("nan")
    flat[4::11] = float("-inf")
    x = _cl(x.to(torch.bfloat16))
    scale = torch.ones(c, device=DEV)
    scale[::2] = 2.0 ** -20
    shift = torch.zeros(c, device=DEV)
    res = None
    if with_res:
        res = torch.randn(shape, device=DEV)
        # where the scale is 1 and the shift 0, -x cancels the normalised value exactly
        res = torch.where(torch.arange(k, device=DEV).view(shape) % 3 == 0, -x.float(), res)
        res = _cl(res.to(torch.bfloat16))
    y, mask = _fwd_with_mask(x, res, scale, shift)
    assert torch.equal(X.unpack_relu_bits(mask, shape), y.float() > 0)
    assert not torch.isnan(y.float()).any()


def _make_pair(c, seed):
    from draco_b200.ops.norm import FusedBatchNorm2d
    g = torch.Generator().manual_seed(seed)
    bns = []
    for _ in range(2):
        bn = FusedBatchNorm2d(c).to(DEV)
        with torch.no_grad():
            bn.weight.copy_(torch.rand(c, generator=g) + 0.5)
            bn.bias.copy_(torch.rand(c, generator=g) - 0.5)
        bns.append(bn)
    return bns


def _stats(x):
    """Per-channel mean / invstd in fp32 (what a convolution epilogue would hand over as pending_stats)."""
    xf = x.float().nan_to_num(0.0, 0.0, 0.0)
    mean = xf.mean(dim=(0, 2, 3))
    var = xf.var(dim=(0, 2, 3), unbiased=False)
    return mean.contiguous(), torch.rsqrt(var + 1e-5).contiguous()


def _run_pair(bn2, bn_s, x, s, gy, pair):
    from draco_b200.ops import norm
    xg, sg = x.clone().requires_grad_(True), s.clone().requires_grad_(True)
    bn2.pending_stats = (xg,) + _stats(x)
    bn_s.pending_stats = (sg,) + _stats(s)
    before = norm.backend_counters["fused"]
    if pair:
        y = bn2(xg, residual_bn=(bn_s, sg), relu=True)
    else:
        y = bn2(xg, residual=bn_s(sg), relu=True)
    assert norm.backend_counters["fused"] - before == 2
    y.backward(gy)
    torch.cuda.synchronize()
    out = [y.detach(), xg.grad, sg.grad, bn2.weight.grad, bn2.bias.grad, bn_s.weight.grad, bn_s.bias.grad,
           bn2.num_batches_tracked.clone(), bn_s.num_batches_tracked.clone()]
    return [t.clone() for t in out]


@pytest.mark.parametrize("shape", [(128, 128, 16, 16), (128, 512, 4, 4), (16, 64, 8, 8), (5, 8, 3, 3), (3, 8, 5, 7),
                                   (2, 2048, 2, 3), (7, 64, 9, 11)])
@pytest.mark.parametrize("special", [False, True])
def test_pair_equals_two_layer_path(shape, special, monkeypatch):
    """One-pass pair relu(bn2(x) + bn_s(s)) vs the saved-output-mask path with two calls: forward, every gradient and the
    batch counters bit-identical, including shortcut inputs with NaN / Inf."""
    from draco_b200.ops import norm
    torch.manual_seed(sum(shape) + special)
    x = _cl((torch.randn(shape, device=DEV) * 1.3 + 0.2).to(torch.bfloat16))
    s = torch.randn(shape, device=DEV)
    if special:
        s.view(-1)[::97] = float("nan")
        s.view(-1)[5::101] = float("inf")
        s.view(-1)[9::103] = float("-inf")
    s = _cl(s.to(torch.bfloat16))
    gy = _cl(torch.randn(shape, device=DEV).to(torch.bfloat16))
    res = {}
    for pair in (False, True):
        monkeypatch.setenv("DRACO_BN_MASK", "bits" if pair else "y")
        bn2, bn_s = _make_pair(shape[1], 7)
        res[pair] = _run_pair(bn2, bn_s, x, s, gy, pair)
    for i, (a, b) in enumerate(zip(res[False], res[True])):
        assert _same(a, b), i
    assert norm.backend_counters["fused"] > 0


def _model_step(make, batch, pair, monkeypatch, hw=32):
    """One bf16 channels-last forward + backward; ``pair=False`` restates the parent path: the ReLU mask read from the saved
    output and the downsampling blocks' two BatchNorms as two calls."""
    from draco_b200.ops import norm
    monkeypatch.setenv("DRACO_BN_MASK", "bits" if pair else "y")
    if not pair:
        monkeypatch.setattr(norm.FusedBatchNorm2d, "_pair_ok", lambda *a, **k: False)
    torch.manual_seed(3)
    m = make().to(DEV)
    for mod in m.modules():
        if not isinstance(mod, torch.nn.modules.batchnorm._BatchNorm):
            for p in mod.parameters(recurse=False):
                p.data = p.data.to(torch.bfloat16)
    m = m.to(memory_format=torch.channels_last)
    g = torch.Generator(device=DEV).manual_seed(5)
    xin = _cl(torch.randn(batch, 3, hw, hw, device=DEV, generator=g).to(torch.bfloat16))
    tgt = torch.randint(0, 10, (batch,), device=DEV, generator=g)
    before = dict(norm.backend_counters)
    loss = F.cross_entropy(m(xin).float(), tgt)
    loss.backward()
    torch.cuda.synchronize()
    fused = norm.backend_counters["fused"] - before["fused"]
    bufs = [b.detach().clone() for b in m.buffers()]
    grads = [p.grad.detach().clone() for p in m.parameters()]
    monkeypatch.undo()
    return loss.detach().clone(), grads, bufs, fused


@pytest.mark.parametrize("net,batch", [("ResNet18", 128), ("ResNet50", 16)])
def test_whole_model_bit_identical_to_parent_path(net, batch, monkeypatch):
    from draco_b200 import models
    make = getattr(models, net)
    ref = _model_step(make, batch, False, monkeypatch)
    new = _model_step(make, batch, True, monkeypatch)
    assert _same(ref[0], new[0])
    assert len(ref[1]) == len(new[1]) and all(_same(a, b) for a, b in zip(ref[1], new[1]))
    assert len(ref[2]) == len(new[2]) and all(_same(a, b) for a, b in zip(ref[2], new[2]))   # running statistics, counts
    assert ref[3] == new[3]
    if net == "ResNet18":
        assert new[3] == 20


def test_pair_graph_replay_equals_eager():
    """The pair's forward + backward captured in a CUDA graph and replayed give the eager results bit for bit."""
    shape = (64, 128, 8, 8)
    torch.manual_seed(11)
    x = _cl(torch.randn(shape, device=DEV).to(torch.bfloat16))
    s = _cl(torch.randn(shape, device=DEV).to(torch.bfloat16))
    gy = _cl(torch.randn(shape, device=DEV).to(torch.bfloat16))
    bn2, bn_s = _make_pair(shape[1], 3)
    eager = _run_pair(bn2, bn_s, x, s, gy, True)

    bn2, bn_s = _make_pair(shape[1], 3)
    xg, sg = x.clone().requires_grad_(True), s.clone().requires_grad_(True)
    st_x, st_s = _stats(x), _stats(s)

    def step():
        bn2.pending_stats = (xg,) + st_x
        bn_s.pending_stats = (sg,) + st_s
        y = bn2(xg, residual_bn=(bn_s, sg), relu=True)
        y.backward(gy)
        return y

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    for t in (xg, sg, bn2.weight, bn2.bias, bn_s.weight, bn_s.bias):
        t.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        y = step()
    for _ in range(2):
        graph.replay()
    torch.cuda.synchronize()
    got = [y.detach(), xg.grad, sg.grad, bn2.weight.grad, bn2.bias.grad, bn_s.weight.grad, bn_s.bias.grad]
    for i, (a, b) in enumerate(zip(eager[:7], got)):
        assert _same(a, b), i
