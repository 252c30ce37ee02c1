"""Host C++ natives: locator (N1), codec (N4), ABI of the CUDA library."""
import ctypes as C
import itertools

import numpy as np
import pytest

from draco_b200 import _native as N
from draco_b200.codes import cyclic
from draco_b200.utils import codec


def _locate(E, n, s, tol=1e-6):
    Eh = np.ascontiguousarray(np.stack([E.real, E.imag], -1)).astype(np.float64)
    T = Eh.shape[0]
    v = np.zeros((T, n, 2))
    mask = np.zeros(T, dtype=np.uint32)
    fl = np.zeros(T, dtype=np.int32)
    assert N.host().drc_host_locate(Eh.ctypes.data, T, n, s, tol, v.ctypes.data, mask.ctypes.data, fl.ctypes.data) == 0
    return v[..., 0] + 1j * v[..., 1], mask, fl


@pytest.mark.parametrize("n,s", [(5, 1), (7, 2), (7, 3), (9, 2)])
def test_cpp_locator_matches_numpy_oracle(n, s):
    rng = np.random.RandomState(0)
    c = cyclic.search_w(n, s)
    G = rng.randn(n, 64)
    f = rng.randn(64) + 1.0
    R0 = np.stack([cyclic.encode(c, i, G) for i in range(n)])
    for k in range(s + 1):
        for liars in itertools.islice(itertools.combinations(range(n), k), 12):
            R = R0.copy()
            for l in liars:
                R[l] += -100.0 * (1 + rng.rand(64))
            v, mask, fl = _locate((R @ f)[None], n, s)
            assert fl[0] >= len(liars) and fl[0] <= s
            for l in liars:
                assert not (mask[0] >> l) & 1, "a liar was used for recombination"
            dec = np.real(v[0] @ R)
            assert np.abs(dec - G.sum(0)).max() < 1e-6 * max(1.0, np.abs(G).sum())


def test_cpp_solve_poly_a_is_the_locator_polynomial():
    n, s = 7, 2
    rng = np.random.RandomState(3)
    c = cyclic.search_w(n, s)
    G = rng.randn(n, 32)
    R = np.stack([cyclic.encode(c, i, G) for i in range(n)])
    R[1] += 100.0
    R[4] -= 70.0
    E = R @ (rng.randn(32) + 1.0)
    Eh = np.ascontiguousarray(np.stack([E.real, E.imag], -1))
    alpha = np.zeros((s, 2))
    assert N.host().drc_host_solve_poly_a(Eh.ctypes.data, n, s, alpha.ctypes.data) == 0
    p = cyclic.locator_values(alpha[:, 0] + 1j * alpha[:, 1], n)
    mag = np.abs(p)
    assert set(np.argsort(mag)[:2]) == {1, 4} and mag[[1, 4]].max() < 1e-6 * mag.max()


@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.complex64, np.int32, np.uint8])
@pytest.mark.parametrize("shape", [(0,), (1,), (4097,), (64, 3, 3, 3), (10000,)])
def test_codec_roundtrip(dtype, shape):
    rng = np.random.RandomState(0)
    a = (rng.randn(*shape) * 1e-3).astype(dtype)
    b = codec.decompress(codec.compress(a))
    assert b.dtype == a.dtype and b.shape == a.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def test_codec_compresses_structured_gradients():
    z = np.zeros(100000, dtype=np.float32)
    assert codec.ratio(z) < 0.01
    g = (np.random.RandomState(0).randn(100000) * 1e-3).astype(np.float32)
    assert codec.ratio(g) < 0.97              # sign/exponent plane packs, mantissa planes stay raw
    sparse = g.copy(); sparse[np.random.RandomState(1).rand(100000) < 0.9] = 0
    assert codec.ratio(sparse) <= 1.01
    with pytest.raises(ValueError):
        codec.decompress(b"garbage-not-a-stream-----")


def test_cuda_library_abi_matches_ctypes():
    lib = N.cuda()            # loads without a GPU (static cudart, libcuda resolved lazily)
    for name in ("PushArgs", "OmniArgs", "VoteArgs", "ResolveArgs", "UpdateArgs", "CastArgs", "WaitArgs", "SetFlagArgs",
                 "TensorMeta", "HyperParams", "TileView", "FlagList", "ProjectArgs", "LocateArgs", "GeoMedArgs",
                 "GeoMedPrepArgs", "PairDistArgs", "KrumSelectArgs"):
        assert getattr(lib, "drc_sizeof_" + name)() == C.sizeof(getattr(N, name)), name


# ------------------------------------------------------------------------------------------------ native input pipeline
def test_native_gather_augment_matches_python_reference():
    import torch

    from draco_b200.data import augment_cifar
    from draco_b200.data.loader import gather_augment
    g = torch.Generator().manual_seed(0)
    images = torch.randint(0, 256, (300, 3, 32, 32), dtype=torch.uint8, generator=g)
    labels = torch.randint(0, 10, (300,), generator=g)
    idx = np.random.RandomState(1).randint(0, 300, size=77)
    out = torch.zeros(77, 3, 32, 32, dtype=torch.uint8)
    lab = torch.zeros(77, dtype=torch.int64)
    gather_augment(images, labels, idx, out, lab)                       # plain gather
    assert torch.equal(out, images[torch.from_numpy(idx)]) and torch.equal(lab, labels[torch.from_numpy(idx)])
    for seed in (1, 12345, 2 ** 31 + 5):
        gather_augment(images, labels, idx, out, lab, seed=seed)        # reflect-pad-4 crop + flip, same draws as Python
        ref = augment_cifar(images[torch.from_numpy(idx)], seed)
        assert torch.equal(out, ref), seed
    with pytest.raises(IndexError):
        gather_augment(images, labels, np.array([0, 300]), out[:2], lab[:2])


def test_native_loader_thread_pool_overlapping_jobs():
    import torch

    from draco_b200.data import augment_cifar
    from draco_b200.data.loader import NativeLoader
    g = torch.Generator().manual_seed(3)
    images = torch.randint(0, 256, (512, 1, 28, 28), dtype=torch.uint8, generator=g)      # MNIST-shaped
    labels = torch.randint(0, 10, (512,), generator=g)
    ld = NativeLoader(images, labels, threads=3)
    rs = np.random.RandomState(4)
    jobs = []
    for j in range(24):
        idx = rs.randint(0, 512, size=64)
        out = torch.zeros(64, 1, 28, 28, dtype=torch.uint8)
        lab = torch.zeros(64, dtype=torch.int64)
        seed = None if j % 3 == 0 else 100 + j
        jobs.append((idx, out, lab, seed, ld.submit(idx, out, lab, seed=seed)))
    ld.wait()
    for idx, out, lab, seed, _ in jobs:
        src = images[torch.from_numpy(idx)]
        assert torch.equal(out, src if seed is None else augment_cifar(src, seed))
        assert torch.equal(lab, labels[torch.from_numpy(idx)])
    t = ld.submit(np.array([600]), torch.zeros(1, 1, 28, 28, dtype=torch.uint8), torch.zeros(1, dtype=torch.int64))
    with pytest.raises(IndexError):
        ld.wait(t)
    ld.close()


# ------------------------------------------------------------------------------------------------ tap-table convolution algebra
@pytest.mark.parametrize("ks,stride", [(3, 1), (3, 2), (1, 2), (1, 1)])
def test_conv_tap_tables_reproduce_fprop_and_parity_class_dgrad(ks, stride):
    """The host-side tables that drive the tap-table wgmma convolutions (csrc/cuda/conv_tap_wgmma.cu), checked by
    emulating the kernel's loads on the CPU: input pixel = patch origin * in_mul + tap offset (out-of-range reads as zero, as
    the TMA unit fills), one weight column block per tap; strided dgrad assembled from its parity classes."""
    import torch
    import torch.nn.functional as F
    if not N.cuda_available():
        pytest.skip("libdraco_cuda.so not built")
    lib = N.cuda()
    lib.drc_convg_taps.argtypes = [C.c_int] * 5 + [C.POINTER(C.c_int)] * 3
    lib.drc_convg_taps.restype = C.c_int

    def taps(dgrad, ph=0, pw=0):
        dh, dw, ti = (C.c_int * 9)(), (C.c_int * 9)(), (C.c_int * 9)()
        n = lib.drc_convg_taps(ks, stride, int(dgrad), ph, pw, dh, dw, ti)
        return [(dh[i], dw[i], ti[i]) for i in range(n)]

    torch.manual_seed(ks * 10 + stride)
    n, cin, cout, H = 2, 4, 5, 8
    pad, OH = ks // 2, H // stride
    x = torch.randn(n, H, H, cin, dtype=torch.float64)                       # NHWC like the kernels
    w = torch.randn(cout, ks, ks, cin, dtype=torch.float64)                  # arena layout [Cout, ks, ks, Cin]
    Wm = w.reshape(cout, ks * ks * cin)

    def gather(t, i0, j0, mul, dh, dw):                                       # t[n, i*mul + dh, j*mul + dw, :] with zero fill
        Hh = t.shape[1]
        out = torch.zeros(n, len(i0), len(j0), t.shape[3], dtype=t.dtype)
        for a_, i in enumerate(i0):
            for b_, j in enumerate(j0):
                hh, ww = i * mul + dh, j * mul + dw
                if 0 <= hh < Hh and 0 <= ww < Hh:
                    out[:, a_, b_] = t[:, hh, ww]
        return out

    # fprop
    y = torch.zeros(n, OH, OH, cout, dtype=torch.float64)
    tt = taps(False)
    assert len(tt) == ks * ks
    for dh, dw, ti in tt:
        y += gather(x, range(OH), range(OH), stride, dh, dw) @ Wm[:, ti * cin:(ti + 1) * cin].t()
    ref = F.conv2d(x.permute(0, 3, 1, 2), w.permute(0, 3, 1, 2), stride=stride, padding=pad).permute(0, 2, 3, 1)
    assert torch.allclose(y, ref, atol=1e-10)

    # dgrad from parity classes (unit-stride reads of dy, stride-s writes of dx)
    dy = torch.randn(n, OH, OH, cout, dtype=torch.float64)
    dx = torch.zeros(n, H, H, cin, dtype=torch.float64)                       # (the launcher zero-fills when a class is empty)
    total = 0
    for ph in range(stride):
        for pw in range(stride):
            tt = taps(True, ph, pw)
            total += len(tt)
            acc = torch.zeros(n, OH, OH, cin, dtype=torch.float64)
            for dh, dw, ti in tt:
                acc += gather(dy, range(OH), range(OH), 1, dh, dw) @ Wm[:, ti * cin:(ti + 1) * cin]
            if tt:
                dx[:, ph::stride, pw::stride] = acc
    assert total == ks * ks                                                   # every filter tap used exactly once overall
    dref = torch.nn.grad.conv2d_input((n, cin, H, H), w.permute(0, 3, 1, 2), dy.permute(0, 3, 1, 2), stride=stride,
                                      padding=pad).permute(0, 2, 3, 1)
    assert torch.allclose(dx, dref, atol=1e-10)


def test_tap_convolution_launch_plans(monkeypatch):
    """Host-side planning of the tap convolution (drc_convg_plan): one CTA per tile by default (the multicast-cluster variant is
    opt-in), a forced shape needs two real tiles along each dimension it multicasts over, grids are whole clusters within the SM
    count (132 on an H100 SXM)."""
    if not N.cuda_available():
        pytest.skip("libdraco_cuda.so not built")
    from draco_b200.ops.conv import convg_plan
    monkeypatch.delenv("DRACO_CONV_CLUSTER", raising=False)
    layers = [(128, 16, 16, 128, 128, 3, 1), (128, 8, 8, 256, 256, 3, 1), (128, 4, 4, 512, 512, 3, 1), (128, 32, 32, 64, 128, 3, 2),
              (32, 56, 56, 64, 64, 3, 1), (32, 14, 14, 256, 256, 3, 1)]
    for (n, h, w, cin, cout, ks, st) in layers:
        for dgrad in (0, 1):
            bn, cm, cn, grid, mode = convg_plan(n, h, w, cin, cout, ks, st, dgrad)
            assert (cm, cn, mode) == (1, 1, 0) and 0 < grid <= 132
            assert bn == (128 if (cin if dgrad else cout) >= 128 else 64)
    monkeypatch.setenv("DRACO_CONV_CLUSTER", "2,2,128")
    bn, cm, cn, grid, mode = convg_plan(128, 8, 8, 256, 256, 3, 1, 1)
    assert (bn, cm, cn, mode) == (128, 2, 2, 1) and grid % 4 == 0
    monkeypatch.setenv("DRACO_CONV_CLUSTER", "1,4,128")          # 128 output channels = one N tile: cn = 4 is not realisable
    assert convg_plan(128, 16, 16, 128, 128, 3, 1, 0)[1:3] != [1, 4]
    assert convg_plan(128, 15, 16, 128, 128, 3, 3, 0) is None     # unsupported geometry
