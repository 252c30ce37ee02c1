"""The fused PS update (aggregate_update_kernel: gradient sources 0 / 1 / 2, the shared SGD / Adam / AMSGrad tail, the unicast
broadcast and the flags), cast_params_kernel and the cyclic decode in front of mode 1 (push encode, cyclic_project, the device
locator), bit for bit against the fp32 / fp64 restatements of tests/exact_ref.py.  Every launch gets its own counters, and every
failure names the tensor, the element and the field."""
import ctypes as C

import numpy as np
import pytest
import torch

import exact_ref as X
from draco_b200 import JobConfig
from draco_b200 import _native as N
from draco_b200.codes import cyclic
from draco_b200.models import build_model
from draco_b200.parallel.arena import ArenaLayout
from draco_b200.parallel.ps import hyperparams_tensor

pytestmark = pytest.mark.gpu

SPECIALS = np.array([0.0, -0.0, 2.0 ** -149, -2.0 ** -149, 1e-39, -3e-39, 3e38, -3e38, np.inf, -np.inf, np.nan], np.float32)


@pytest.fixture(scope="module")
def K():
    from draco_b200.ops import kernels
    return kernels


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def lenet():
    """8 tensors, most ending mid-tile (500, 20, 25000, ... elements)."""
    return ArenaLayout.from_model(build_model("LeNet"), bf16=False, channels_last=True)


@pytest.fixture(scope="module")
def resnet():
    return ArenaLayout.from_model(build_model("ResNet18"), bf16=True, channels_last=True)


def ctrl(dev, step):
    """Fresh step counter, done counter and 16 flags for one launch."""
    return (torch.full((1,), step, dtype=torch.int64, device=dev), torch.zeros(1, dtype=torch.int32, device=dev),
            torch.zeros(16, dtype=torch.int64, device=dev))


def valid_mask(L, dev=None):
    m = torch.from_numpy(L.valid_mask())
    return m if dev is None else m.to(dev)


def edge_rows(L, rows, seed, dev, scale=0.5, p_special=0.02):
    """fp32 [rows, total] on the device: N(0, scale^2) with a fraction p_special of +-0, +-subnormals, +-3e38 (sums overflow),
    +-Inf and NaN; padding +0."""
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(rows, L.total, generator=g, device=dev) * scale
    sp = torch.from_numpy(SPECIALS).to(dev)
    pick = torch.rand(rows, L.total, generator=g, device=dev) < p_special
    which = torch.randint(0, len(SPECIALS), (rows, L.total), generator=g, device=dev)
    x = torch.where(pick, sp[which], x)
    return torch.where(valid_mask(L, dev), x, torch.zeros((), device=dev))


def sample_elems(L, dense: bool, seed=0):
    """Element indices checked on the host, per tensor: every element (dense), or the first and the last tile of each tensor
    plus one tile in between (the tail tile ends mid-tile)."""
    rng = np.random.default_rng(seed)
    out = []
    for sp in L.specs:
        if dense:
            out.append(np.arange(sp.offset, sp.offset + sp.numel))
            continue
        nt = -(-sp.numel // 1024)
        qs = sorted({0, nt - 1, int(rng.integers(0, nt))})
        idx = np.concatenate([sp.offset + q * 1024 + np.arange(min(1024, sp.numel - q * 1024)) for q in qs])
        out.append(idx)
    return out


def first_diff(field, t, idx, got, want):
    """'' if got equals want bit for bit (NaN matches NaN), else the field, tensor and element of the first difference."""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    bad = (got.view(np.uint32) != want.view(np.uint32)) & ~(np.isnan(got) & np.isnan(want))
    if not bad.any():
        return ""
    j = int(np.nonzero(bad)[0][0])
    return (f"{field}: tensor {t}, arena element {int(idx[j])}: got {got[j]!r} "
            f"({got[j:j+1].view(np.uint32)[0]:#010x}), expected {want[j]!r} ({want[j:j+1].view(np.uint32)[0]:#010x}); "
            f"{int(bad.sum())} of {bad.size} differ")


def assert_fields(checks):
    msgs = [m for m in (first_diff(*c) for c in checks) if m]
    assert not msgs, "\n".join(msgs)


def host(t, idx):
    return t.detach().cpu().numpy()[..., idx] if t.dim() == 1 else t.detach().cpu().numpy()[:, idx]


# ------------------------------------------------------------------------------------------------------------------------------
# gradient sources
# ------------------------------------------------------------------------------------------------------------------------------
SGD_PLAIN = dict(lr=0.1, momentum=0.9, weight_decay=5e-4)


def _run_source(K, L, dev, mode, Krows, with_select, seed, dense):
    P = Krows + 2
    rows = edge_rows(L, P, seed, dev)
    rng = np.random.default_rng(seed)
    T = L.ntensors
    sel = torch.from_numpy(rng.integers(0, P, (Krows, T)).astype(np.int32)).to(dev) if with_select else None
    wts = None
    if mode == 2:
        w = rng.standard_normal((T, Krows)).astype(np.float32)
        w[rng.random((T, Krows)) < 0.2] = 0.0
        wts = torch.from_numpy(w).to(dev)
    scale = 1.0 / Krows if mode == 0 else 1.0
    params = edge_rows(L, 1, seed + 1, dev, p_special=0.0)[0]
    mom = edge_rows(L, 1, seed + 2, dev, scale=0.01, p_special=0.0)[0]
    p0, m0 = params.clone(), mom.clone()
    gout = torch.full((L.total,), 7.0, device=dev)
    hp = hyperparams_tensor(JobConfig(**SGD_PLAIN), dev)
    step, cnt, _ = ctrl(dev, 3)
    K.aggregate_update(L, rows, L.total, params=params, momentum=mom, hp=hp, step_ptr=step, done_counter=cnt, K=Krows,
                       scale=scale, select=sel, weights=wts, first_step=1, grad_out=gout)
    torch.cuda.synchronize()
    selh = sel.cpu().numpy() if with_select else None
    elems = sample_elems(L, dense, seed)
    cat = torch.from_numpy(np.concatenate(elems)).to(dev)
    rows_h, p0_h, m0_h, gout_h, p_h, m_h = (a[..., cat].cpu().numpy() for a in (rows, p0, m0, gout, params, mom))
    checks, at = [], 0
    for t, idx in enumerate(elems):
        sl = slice(at, at + len(idx))
        at += len(idx)
        slots = selh[:, t] if with_select else np.arange(Krows)
        g = X.update_source_ref(mode, rows_h[slots][:, sl], np.float32(scale), weights=None if wts is None else w[t])
        p, m = X.sgd_tail_ref(g, p0_h[sl], m0_h[sl], dampening=0.0, nesterov=False, first=False, **SGD_PLAIN)
        checks += [("grad_out", t, idx, gout_h[sl], g), ("params", t, idx, p_h[sl], p), ("momentum", t, idx, m_h[sl], m)]
    assert_fields(checks)
    return gout, params


@pytest.mark.parametrize("Krows", [1, 2, 3, 7, 16, 32])
@pytest.mark.parametrize("with_select", [False, True])
def test_mode0_select_sum_lenet(K, dev, lenet, Krows, with_select):
    """Mode 0 (mean, vote winners): the K rows summed from +0 in ascending k, one rounded multiply by fp32(1/K)."""
    _run_source(K, lenet, dev, 0, Krows, with_select, 100 + Krows, dense=True)


@pytest.mark.parametrize("Krows", [1, 2, 3, 7, 16])
@pytest.mark.parametrize("with_select", [False, True])
def test_mode2_weights_lenet(K, dev, lenet, Krows, with_select):
    """Mode 2 (geometric median, Krum folds): an fmaf chain over the K rows in order, zero weights included."""
    _run_source(K, lenet, dev, 2, Krows, with_select, 200 + Krows, dense=True)


@pytest.mark.parametrize("mode,Krows", [(0, 3), (0, 32), (2, 16)])
def test_sources_resnet18(K, dev, resnet, mode, Krows):
    """The same on the ResNet-18 arena (62 tensors, 11.2 M elements), checked on three tiles of every tensor."""
    _run_source(K, resnet, dev, mode, Krows, True, 300 + Krows, dense=False)


# ------------------------------------------------------------------------------------------------------------------------------
# SGD tail
# ------------------------------------------------------------------------------------------------------------------------------
SGD_CASES = [(mu, damp, wd, nest) for mu in (0.0, 0.9) for damp in (0.0, 0.1, 0.5) for wd in (0.0, 5e-4)
             for nest in (False, True) if not (nest and (damp != 0 or mu == 0))]


@pytest.mark.parametrize("mu,damp,wd,nest", SGD_CASES)
def test_sgd_tail_first_and_later_steps(K, dev, lenet, mu, damp, wd, nest):
    """Weight decay, the first-step copy (no dampening), dampening with fp32(1 - dampening) formed in fp64, and Nesterov:
    params and momentum bit-exact on the first step and on two later ones (first_step = 4)."""
    L = lenet
    hpd = dict(lr=0.05, momentum=mu, weight_decay=wd, dampening=damp, nesterov=nest)
    hp = hyperparams_tensor(JobConfig(**hpd), dev)
    params = edge_rows(L, 1, 11, dev, p_special=0.0)[0]
    mom = edge_rows(L, 1, 12, dev, scale=0.01, p_special=0.0)[0]
    idx = np.arange(L.total)
    p, m = host(params, idx), host(mom, idx)
    for it, stepv in enumerate((4, 5, 6)):
        rows = edge_rows(L, 3, 20 + it, dev, scale=0.3, p_special=0.001)
        step, cnt, _ = ctrl(dev, stepv)
        gout = torch.zeros(L.total, device=dev)
        K.aggregate_update(L, rows, L.total, params=params, momentum=mom, hp=hp, step_ptr=step, done_counter=cnt, K=3,
                           scale=1.0 / 3, first_step=4, grad_out=gout)
        torch.cuda.synchronize()
        g = X.update_source_ref(0, host(rows, idx), np.float32(1.0 / 3))
        p, m = X.sgd_tail_ref(g, p, m, first=stepv == 4, **hpd)
        assert_fields([("grad_out", "all", idx, host(gout, idx), g), (f"params (step {stepv})", "all", idx, host(params, idx), p),
                       (f"momentum (step {stepv})", "all", idx, host(mom, idx), m)])


def test_sgd_50_step_chain_is_bit_exact(K, dev, lenet):
    """50 steps of Nesterov SGD with weight decay: params and momentum equal the restatement bit for bit after every step."""
    L = lenet
    hpd = dict(lr=0.05, momentum=0.9, weight_decay=5e-4, dampening=0.0, nesterov=True)
    hp = hyperparams_tensor(JobConfig(**hpd), dev)
    params = edge_rows(L, 1, 31, dev, p_special=0.0)[0]
    mom = torch.zeros(L.total, device=dev)
    idx = np.arange(L.total)
    p, m = host(params, idx), host(mom, idx)
    step, cnt, _ = ctrl(dev, 1)
    for it in range(1, 51):
        rows = edge_rows(L, 4, 1000 + it, dev, scale=0.3, p_special=0.0)
        step.fill_(it)
        K.aggregate_update(L, rows, L.total, params=params, momentum=mom, hp=hp, step_ptr=step, done_counter=cnt, K=4,
                           scale=0.25, first_step=1)
        g = X.update_source_ref(0, host(rows, idx), np.float32(0.25))
        p, m = X.sgd_tail_ref(g, p, m, first=it == 1, **hpd)
        assert_fields([(f"params (step {it})", "all", idx, host(params, idx), p),
                       (f"momentum (step {it})", "all", idx, host(mom, idx), m)])
    assert int(cnt.item()) == 0


# ------------------------------------------------------------------------------------------------------------------------------
# Adam / AMSGrad tail
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("amsgrad", [False, True])
@pytest.mark.parametrize("t", [1, 2, 3, 10, 1000, 100000])
def test_adam_tail_bit_exact(K, dev, lenet, amsgrad, t):
    """One Adam / AMSGrad step at update count t, set through step_ptr with first_step = 7 (a resumed job), from a random
    state with v = 0 in places, vmax below and above v, and gradients whose square overflows (|g| ~ 1e20..1e30) or underflows
    (|g| ~ 1e-25): params, exp_avg, exp_avg_sq and max_exp_avg_sq bit-exact."""
    L = lenet
    first_step = 7
    cfg = JobConfig(optimizer="adam", amsgrad=amsgrad, lr=1e-3, weight_decay=1e-4)
    hp = hyperparams_tensor(cfg, dev)
    rng = np.random.default_rng(t)
    n = L.total
    mask = L.valid_mask()
    p0 = (rng.standard_normal(n) * np.where(rng.random(n) < 0.5, 1e-4, 1.0)).astype(np.float32)
    m0 = (rng.standard_normal(n) * 0.01).astype(np.float32)
    v0 = (rng.random(n) * 1e-3).astype(np.float32)
    v0[rng.random(n) < 0.1] = 0.0
    vm0 = (v0 * rng.choice([0.5, 1.0, 2.0], n)).astype(np.float32)
    g = (rng.standard_normal((2, n)) * 0.1).astype(np.float32)
    big, tiny = rng.random(n) < 0.01, rng.random(n) < 0.01
    g[0, big] = (rng.standard_normal(big.sum()) * 10.0 ** rng.uniform(20, 30, big.sum())).astype(np.float32)
    g[0, tiny] = (rng.standard_normal(tiny.sum()) * 1e-25).astype(np.float32)
    p0, m0, v0, vm0 = (np.where(mask, a, np.float32(0)) for a in (p0, m0, v0, vm0))
    g = np.where(mask, g, np.float32(0))
    dv = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    params, mom, v, vm, rows = dv(p0), dv(m0), dv(v0), dv(vm0), dv(g)
    step, cnt, _ = ctrl(dev, first_step + t - 1)
    K.aggregate_update(L, rows, n, params=params, momentum=mom, exp_avg_sq=v, max_exp_avg_sq=vm if amsgrad else None, hp=hp,
                       step_ptr=step, done_counter=cnt, K=2, scale=0.5, first_step=first_step)
    torch.cuda.synchronize()
    gr = X.update_source_ref(0, g, np.float32(0.5))
    a = X.adam_step_size_ref(1e-3, 0.9, 0.999, first_step + t - 1, first_step)
    p, m, vv, vmm = X.adam_tail_ref(gr, p0, m0, v0, vm0, step_size=a, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=1e-4,
                                    amsgrad=amsgrad)
    idx = np.arange(n)
    checks = [("params", "all", idx, host(params, idx), p), ("momentum", "all", idx, host(mom, idx), m),
              ("exp_avg_sq", "all", idx, host(v, idx), vv)]
    if amsgrad:
        checks.append(("max_exp_avg_sq", "all", idx, host(vm, idx), vmm))
    assert_fields(checks)
    assert np.isinf(vv).any()                                                       # d * d overflowed somewhere


# ------------------------------------------------------------------------------------------------------------------------------
# broadcast, flags, launch shape, padding
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("opt", ["sgd", "amsgrad"])
def test_broadcast_flags_grids_buckets_and_padding(K, dev, resnet, opt):
    """0, 1 and 16 unicast destinations each equal params; the flags end at step + 1 and done_counter returns to 0; grids
    1, 7, the SM count and 1000 and a 3-bucket tile split give identical bits; padding stays +0 in every arena."""
    L = resnet
    cfg = JobConfig(**SGD_PLAIN) if opt == "sgd" else JobConfig(optimizer="adam", amsgrad=True, lr=1e-3)
    hp = hyperparams_tensor(cfg, dev)
    rows = edge_rows(L, 3, 41, dev, p_special=0.0)
    p_init = edge_rows(L, 1, 42, dev, p_special=0.0)[0]
    pad = ~valid_mask(L, dev)
    results = []
    shapes = [dict(grid=g) for g in (1, 7, K.sm_count(), 1000)] + [dict(buckets=3)]
    for i, shape in enumerate(shapes):
        params, mom = p_init.clone(), torch.zeros(L.total, device=dev)
        v = torch.zeros(L.total, device=dev) if opt != "sgd" else None
        vm = torch.zeros(L.total, device=dev) if opt != "sgd" else None
        ndst = (0, 1, 16)[i % 3]
        dst = [torch.full((L.total,), 5.0, device=dev) for _ in range(ndst)]
        gout = torch.full((L.total,), 9.0, device=dev)
        step, cnt, flags = ctrl(dev, 11)
        kw = dict(params=params, momentum=mom, exp_avg_sq=v, max_exp_avg_sq=vm, hp=hp, step_ptr=step, done_counter=cnt, K=3,
                  scale=1.0 / 3, first_step=11, grad_out=gout, dst=dst, flags=[flags[j:j + 1] for j in (0, 3, 15)])
        if "buckets" in shape:
            cuts = [0, L.ntiles // 3, 2 * L.ntiles // 3, L.ntiles]
            for b in range(3):
                K.aggregate_update(L, rows, L.total, tile_range=(cuts[b], cuts[b + 1]), **kw)
        else:
            K.aggregate_update(L, rows, L.total, grid=shape["grid"], **kw)
        torch.cuda.synchronize()
        for j, d in enumerate(dst):
            assert torch.equal(d.view(torch.int32), params.view(torch.int32)), f"{shape}: destination {j} differs from params"
        fl = flags.tolist()
        assert [fl[0], fl[3], fl[15]] == [12, 12, 12] and sum(fl) == 36, f"{shape}: flags {fl}"
        assert int(cnt.item()) == 0, f"{shape}: done_counter {int(cnt.item())}"
        for name, a in (("params", params), ("momentum", mom), ("grad_out", gout), ("exp_avg_sq", v), ("max_exp_avg_sq", vm)):
            if a is not None:
                assert int(a[pad].view(torch.int32).abs().sum()) == 0, f"{shape}: padding of {name} is not +0"
        results.append([a.view(torch.int32).clone() for a in (params, mom, gout) + ((v, vm) if v is not None else ())])
    for shape, r in zip(shapes[1:], results[1:]):
        for name, a, b in zip(("params", "momentum", "grad_out", "exp_avg_sq", "max_exp_avg_sq"), r, results[0]):
            assert torch.equal(a, b), f"{name}: {shape} differs from grid 1"


# ------------------------------------------------------------------------------------------------------------------------------
# cast_params
# ------------------------------------------------------------------------------------------------------------------------------
def test_cast_params_rne_bit_exact(K, dev, resnet):
    """bf16 tensors: round to nearest even on ties, subnormals, values that round to +-Inf and +-0, NaN stays NaN; the fp32
    tensors' part of the bf16 arena is not written."""
    L = resnet
    rng = np.random.default_rng(51)
    n = L.total
    x = (rng.standard_normal(n) * 2.0).astype(np.float32)
    u = x.view(np.uint32)
    k = rng.random(n)
    u[k < 0.05] = (u[k < 0.05] & 0xFFFF0000) | 0x8000                                   # exact ties, even and odd
    e = rng.random(n) < 0.05
    x[e] = rng.choice(np.array([2.0 ** -149, -2.0 ** -140, 1e-39, 3.3961e38, -3.3961e38, 3.4e38, 0.0, -0.0, np.inf, np.nan,
                                np.float32(3.38953139e38)], np.float32), e.sum())
    x = np.where(L.valid_mask(), x, np.float32(0))
    src = torch.from_numpy(x).to(dev)
    dst = torch.full((n,), 0x1234, dtype=torch.int16, device=dev).view(torch.bfloat16)
    K.cast_params(L, src, dst)
    torch.cuda.synchronize()
    got = dst.view(torch.int16).cpu().numpy().view(np.uint16)
    want = X.cast_bf16_ref(x)
    for t, sp in enumerate(L.specs):
        sl = slice(sp.offset, sp.offset + sp.numel)
        if sp.is_bf16:
            gn = np.isnan(torch.from_numpy(got[sl].view(np.int16)).view(torch.bfloat16).float().numpy())
            nan = np.isnan(x[sl])
            bad = np.nonzero((got[sl] != want[sl]) & ~nan | (nan != gn))[0]
            assert not len(bad), (f"bf16 params: tensor {t}, element {sp.offset + bad[0]}: x = {x[sl][bad[0]]!r}, "
                                  f"got {got[sl][bad[0]]:#06x}, expected {want[sl][bad[0]]:#06x}; {len(bad)} differ")
        else:
            assert (got[sl] == 0x1234).all(), f"bf16 arena: fp32 tensor {t} was written"


# ------------------------------------------------------------------------------------------------------------------------------
# cyclic chain: push encode -> cyclic_project -> locator -> mode 1
# ------------------------------------------------------------------------------------------------------------------------------
def tile_tables(L):
    tt, valid = np.zeros(L.ntiles, np.int64), np.zeros(L.ntiles, np.int64)
    for t, sp in enumerate(L.specs):
        nt = -(-sp.numel // 1024)
        q = np.arange(nt)
        tt[sp.offset // 1024 + q] = t
        valid[sp.offset // 1024 + q] = np.minimum(1024, sp.numel - 1024 * q)
    return tt, valid


def encode_ref(code, w, G, attack, mag, mask):
    """push_encode_kernel's cyclic path for worker w: re / im = fmaf chains over its r batches (fp32 coefficients), then for a
    liar, rev_grad re = rn(re + rn(mag * re)) and im = fma(im, mag, im), constant re = rn(re + mag) on real elements."""
    co = code.coeffs_of(w).astype(np.complex64)
    re = im = np.zeros(G.shape[1], np.float32)
    for k, b in enumerate(code.batches_of(w)):
        re = X._fma32(co[k].real, G[b], re)
        im = X._fma32(co[k].imag, G[b], im)
    if attack == 1:
        re = X._add32(re, np.where(mask, X._mul32(np.float32(mag), re), np.float32(0)))
        im = X._fma32(im, np.float32(mag), im)
    elif attack == 2:
        re = X._add32(re, np.where(mask, np.float32(mag), np.float32(0)))
    return re, im


@pytest.mark.parametrize("n,s", [(3, 1), (5, 2), (7, 3), (8, 3), (9, 3), (15, 3), (16, 2), (17, 3), (31, 3), (32, 3)])
def test_cyclic_chain_bit_exact(K, dev, lenet, n, s):
    L = lenet
    code = cyclic.search_w(n, s)
    rng = np.random.default_rng(n * 10 + s)
    liars = sorted({n - 1} | set(rng.choice(n - 1, s - 1, replace=False).tolist()))
    mask = L.valid_mask()
    G = np.where(mask, rng.standard_normal((n, L.total)) * 0.05, 0).astype(np.float32)
    Gd = torch.from_numpy(G).to(dev)
    R = torch.zeros(n, 2 * L.total, device=dev)
    bitmap = torch.from_numpy(np.array([sum(1 << q for q in liars)], np.uint32).view(np.int32)).to(dev)   # slot 31: bit 31
    step, cnt, _ = ctrl(dev, 1)
    attack_of = {q: 1 + (j % 2) for j, q in enumerate(liars)}                            # rev_grad, constant, ...
    for w in range(n):
        b = code.batches_of(w)
        K.push_encode(L, [Gd[j] for j in b], [None] * len(b), R[w], step_ptr=step, worker=w, done_counter=cnt,
                      coef=list(code.coeffs_of(w)), adv_bitmap=bitmap, adv_len=1, attack=attack_of.get(w, 1), magnitude=-100.0)
    # the random attack: only its padding is specified (zero)
    Rrand = torch.full((2 * L.total,), 3.0, device=dev)
    b = code.batches_of(n - 1)
    K.push_encode(L, [Gd[j] for j in b], [None] * len(b), Rrand, step_ptr=step, worker=n - 1, done_counter=cnt,
                  coef=list(code.coeffs_of(n - 1)), adv_bitmap=bitmap, adv_len=1, attack=3, magnitude=-100.0)
    torch.cuda.synchronize()
    Rh = R.cpu().numpy().reshape(n, L.total, 2)
    Rre, Rim = np.ascontiguousarray(Rh[..., 0]), np.ascontiguousarray(Rh[..., 1])
    assert (Rrand.cpu().numpy().reshape(L.total, 2)[~mask] == 0).all(), "random attack: padding of the codeword is not zero"
    idx = np.arange(L.total)
    for w in range(n):
        re, im = encode_ref(code, w, G, attack_of.get(w, 0), -100.0, mask)
        assert_fields([(f"push encode re (worker {w}{', liar' if w in liars else ''})", "all", idx, Rre[w], re),
                       (f"push encode im (worker {w}{', liar' if w in liars else ''})", "all", idx, Rim[w], im)])
    # projection E = R f per tensor
    f = np.where(mask, rng.standard_normal(L.total) + 1.0, 0).astype(np.float32)
    T = L.ntensors
    E = torch.zeros(T, n, 2, dtype=torch.float64, device=dev)
    K.cyclic_project(L, R, L.total, n, torch.from_numpy(f).to(dev), E)
    torch.cuda.synchronize()
    tt, valid = tile_tables(L)
    Er, Ei = X.cyclic_project_ref(Rre, Rim, f, tt, valid)
    Eh = E.cpu().numpy()
    for t in range(T):
        for i in range(n):
            assert Eh[t, i, 0] == Er[t, i] and Eh[t, i, 1] == Ei[t, i], \
                f"E: tensor {t}, worker {i}: got {tuple(Eh[t, i])}, expected {(Er[t, i], Ei[t, i])}"
    # locator: device against the host build of the same core, on the same E
    recomb = torch.zeros(T, n, 2, dtype=torch.float32, device=dev)
    healthy = torch.zeros(T, dtype=torch.int32, device=dev)
    flagged = torch.zeros(T, dtype=torch.int32, device=dev)
    K.cyclic_locate(E, n, s, recomb, healthy, flagged, rel_tol=1e-4)
    E64 = np.ascontiguousarray(Eh)
    v_host = np.zeros((T, n, 2))
    h_host, f_host = np.zeros(T, np.uint32), np.zeros(T, np.int32)
    rc = N.host().drc_host_locate(E64.ctypes.data, T, n, s, C.c_double(1e-4), v_host.ctypes.data, h_host.ctypes.data,
                                  f_host.ctypes.data)
    assert rc == 0
    torch.cuda.synchronize()
    hd, fd = healthy.cpu().numpy().astype(np.uint32), flagged.cpu().numpy()
    liar_bits = sum(1 << q for q in liars)
    for t in range(T):
        assert hd[t] == h_host[t] and fd[t] == f_host[t], f"tensor {t}: device healthy {hd[t]:#x} / flagged {fd[t]}, host " \
                                                           f"{h_host[t]:#x} / {f_host[t]}"
        assert fd[t] == len(liars) and not (int(hd[t]) & liar_bits), f"tensor {t}: healthy {hd[t]:#x}, liars {liars}"
    vd = recomb.cpu().numpy()
    # the device and the host run the same fp64 locator, compiled differently (FMA contraction): they may differ in the
    # last fp64 bits, which the solve amplifies by its conditioning; bound: 2^-16 of the largest |v| of the tensor
    rel = np.abs(vd - v_host).max(axis=(1, 2)) / np.abs(v_host).max(axis=(1, 2))
    print(f"n={n} s={s}: worst |v_dev - v_host| / max |v_host| = {rel.max():.3e}")
    assert (rel <= 2.0 ** -16).all(), f"recomb: tensor {int(rel.argmax())} differs from the host by {rel.max():.3e}"
    assert (vd[:, liars] == 0).all(), "recomb: a flagged row has a nonzero coefficient"
    # mode 1 on the device's recomb
    hp = hyperparams_tensor(JobConfig(lr=1.0, momentum=0.0), dev)
    params = torch.zeros(L.total, device=dev)
    mom = torch.zeros(L.total, device=dev)
    gout = torch.zeros(L.total, device=dev)
    step2, cnt2, _ = ctrl(dev, 1)
    K.aggregate_update(L, R, L.total, params=params, momentum=mom, hp=hp, step_ptr=step2, done_counter=cnt2, K=n,
                       scale=1.0 / n, recomb=recomb, grad_out=gout)
    torch.cuda.synchronize()
    gh = gout.cpu().numpy()
    vc = vd[..., 0] + 1j * vd[..., 1]
    checks = []
    # decoded gradient against the fp64 mean.  dec = sum_k (1/n + eps_k) g_k + rounding, eps_k = Re(sum_i v_i c_ik) / n - 1/n
    # from the fp32 v and c actually used; rounding <= (r + n + 3) 2^-24 A with A = (1/n) sum_i |v_i|_1 sum_k |c_ik|_1 |g_k|
    # (r fmas of the encode, two roundings per row and n adds of the recombination, the scale), doubled
    W = np.zeros((n, n), np.complex128)
    for i in range(n):
        W[i, code.batches_of(i)] = code.coeffs_of(i).astype(np.complex64)
    worst = 0.0
    for t, sp in enumerate(L.specs):
        sl = np.arange(sp.offset, sp.offset + sp.numel)
        checks.append(("grad_out (mode 1)", t, sl, gh[sl],
                       X.update_source_ref(1, (Rre[:, sl], Rim[:, sl]), np.float32(1.0 / n), recomb=vc[t].astype(np.complex64))))
        Gt = G[:, sl].astype(np.float64)
        mean = Gt.mean(0)
        eps_k = (vc[t].astype(np.complex128) @ W).real / n - 1.0 / n
        v1 = np.abs(vc[t].real) + np.abs(vc[t].imag)
        A = (v1 @ (np.abs(W.real) + np.abs(W.imag)) @ np.abs(Gt)) / n
        bound = np.abs(eps_k) @ np.abs(Gt) + 2 * (code.r + n + 3) * 2.0 ** -24 * A + 2.0 ** -23 * np.abs(mean)
        err = np.abs(gh[sl] - mean)
        assert (err <= bound).all(), f"decoded gradient: tensor {t}, element {int(sl[np.argmax(err - bound)])}: " \
                                     f"|err| {err.max():.3e} outside the bound"
        worst = max(worst, float((err / bound).max()))
    print(f"n={n} s={s}: worst decoded error / bound = {worst:.3f}")
    assert_fields(checks)
