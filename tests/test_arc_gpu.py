"""Adaptive robust clipping (``--arc``) on the GPU: csrc/cuda/arc.cu's factors against the oracle on the LeNet and ResNet-18 arenas
at both scopes, the scale pass bit for bit with padding untouched, grid and bucket independence, the fused PS against the
library-op PS for every rule, graph replay, f = 0, the transport self-check, compression, and training under sign-flip liars."""
import numpy as np
import pytest
import torch

from draco_b200 import JobConfig
from draco_b200.codes import oracle
from draco_b200.models import build_model
from draco_b200.parallel.arena import ArenaLayout
from draco_b200.parallel.trainer import Trainer

pytestmark = pytest.mark.gpu
PAD = 7.0                                         # what the padding holds: the kernels must never write it


@pytest.fixture(scope="module")
def K():
    from draco_b200.ops import kernels
    return kernels


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda", 0)


_LAYOUTS = {}


def _layout(net):
    if net not in _LAYOUTS:
        m = build_model(net) if net == "LeNet" else build_model(net, num_classes=10)
        _LAYOUTS[net] = ArenaLayout.from_model(m, bf16=net == "ResNet18", channels_last=True)
    return _LAYOUTS[net]


def _spans(L):
    return [(s.offset, s.numel) for s in L.specs]


def _slab(L, P, seed):
    """[P, D] fp32 rows whose norms differ per tensor (so each tensor clips other rows), padding = PAD."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(P, L.total, generator=g)
    for sp in L.specs:
        x[:, sp.offset: sp.offset + sp.numel] *= torch.rand(P, 1, generator=g) * 4 + 0.05
    x[:, ~torch.from_numpy(L.valid_mask())] = PAD
    return x


def _ulps(a, b):
    a, b = np.asarray(a, np.float32).view(np.int32).astype(np.int64), np.asarray(b, np.float32).view(np.int32).astype(np.int64)
    return np.abs(a - b)


def _clip(K, L, slab, P, f, scope, dev, **kw):
    ws = K.ArcWorkspace(L, P, dev, model=scope == "model")
    n = K.arc_clip(L, slab, L.total, P, oracle.arc_k(P, f), ws, **kw)
    torch.cuda.synchronize()
    assert n == (4 if scope == "model" else 3)
    return ws


def _check_factors(K, dev, L, S, f, scope):
    P = S.shape[0]
    slab = S.to(dev)
    ws = _clip(K, L, slab, P, f, scope, dev)
    got = ws.factors.cpu().numpy()
    want = oracle.arc_factors(S.numpy(), _spans(L), f, scope)
    assert _ulps(got, want).max() <= 1, (P, scope, _ulps(got, want).max())
    assert np.array_equal(got == 0, want == 0)
    # the scale pass: the fp32 restatement from the kernel's own factors, padding included, bit for bit
    # (NaN compared as NaN: the GPU's multiply returns its one canonical NaN, the host keeps a NaN input's payload)
    ref = oracle.arc(S.numpy(), _spans(L), f, scope, factors=got)
    out = slab.cpu().numpy()
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(out), nan), (P, scope)
    assert np.array_equal(out[~nan].view(np.int32), ref[~nan].view(np.int32)), (P, scope)
    return got


@pytest.mark.parametrize("scope", ["tensor", "model"])
def test_factors_and_scale_on_the_lenet_arena_for_every_worker_count(K, dev, scope):
    L = _layout("LeNet")
    for P in range(1, 17):
        for f in sorted({0, 1, P // 4, (P - 1) // 2}):
            if 0 <= f <= P:
                a = _check_factors(K, dev, L, _slab(L, P, 10 * P + f), f, scope)
                assert (a < 1).sum(1).max() <= oracle.arc_k(P, f)


@pytest.mark.parametrize("scope", ["tensor", "model"])
def test_factors_and_scale_on_the_resnet18_arena(K, dev, scope):
    """Single-tile BatchNorm vectors and 2304-tile 3x3x512x512 convolutions."""
    L = _layout("ResNet18")
    tiles = [-(-sp.numel // 1024) for sp in L.specs]
    assert min(tiles) == 1 and max(tiles) > 2000
    base = _slab(L, 16, 5)
    for P in range(1, 17):
        f = max(0, (P - 1) // 4) if P > 1 else 0
        a = _check_factors(K, dev, L, base[:P].clone(), f, scope)
        if oracle.arc_k(P, f) > 0:
            assert (a < 1).any()


@pytest.mark.parametrize("scope", ["tensor", "model"])
def test_nan_and_inf_rows_match_the_oracle(K, dev, scope):
    L = _layout("LeNet")
    S = _slab(L, 9, 3)
    sp = L.specs[2]
    S[1, sp.offset + 5] = float("nan")
    S[4, sp.offset + 9] = float("inf")
    S[6, L.specs[0].offset] = float("-inf")
    a = _check_factors(K, dev, L, S, 3, scope)                     # k = 4 >= the 3 non-finite rows
    if scope == "tensor":
        assert a[2, 1] == 1 and a[2, 4] == 0 and a[0, 6] == 0
    else:
        assert a[0, 1] == 1 and a[0, 4] == 0 and a[0, 6] == 0
    T = S.clone()
    T[[0, 2, 3], sp.offset] = float("nan")                         # 5 non-finite rows in tensor 2 > k = 4: nothing clips there
    a = _check_factors(K, dev, L, T, 3, scope)
    assert (a[2] == 1).all()


@pytest.mark.parametrize("scope", ["tensor", "model"])
def test_factors_and_slab_do_not_depend_on_the_grid_or_the_bucket_cuts(K, dev, scope):
    L = _layout("ResNet18")
    S = _slab(L, 15, 9).to(dev)
    runs = []
    for grid in (None, 1, 3, 1000):
        slab = S.clone()
        runs.append((_clip(K, L, slab, 15, 3, scope, dev, grid=grid).factors.clone(), slab))
    if scope == "tensor":                                          # whole tensors per bucket, as the pipelined PS cuts them
        T = L.ntensors
        cuts = [0, 3, T // 2, T - 1, T]
        slab = S.clone()
        ws = K.ArcWorkspace(L, 15, dev, model=False)
        for t0, t1 in zip(cuts, cuts[1:]):
            a, b = L.specs[t0].offset // 1024, (L.specs[t1 - 1].offset + L.specs[t1 - 1].numel + 1023) // 1024
            K.arc_clip(L, slab, L.total, 15, 4, ws, tile_range=(a, b), tensor_range=(t0, t1), grid=7)
        torch.cuda.synchronize()
        runs.append((ws.factors.clone(), slab))
    for fa, sl in runs[1:]:
        assert torch.equal(fa, runs[0][0]) and torch.equal(sl.view(torch.int32), runs[0][1].view(torch.int32))


# ------------------------------------------------------------------------------------------------ engine
def _cfg(**kw):
    base = dict(network="LeNet", dataset="MNIST", batch_size=16, max_steps=12, num_workers=7, transport="nvl", lr=0.02,
                momentum=0.9, synthetic_size=512, eval_freq=10 ** 6, compress_grad="None", dtype="fp32", cuda_graphs=False,
                approach="baseline", worker_fail=1, err_mode="constant")
    base.update(kw)
    return JobConfig(**base)


def _run(cfg, steps):
    t = Trainer(cfg, rank=0, world=1, device=torch.device("cuda", 0), quiet=True)
    losses = [t.train_step()["loss"] for _ in range(steps)]
    t.synchronize()
    return t, losses


# the rules of the fused-against-library-op checks; the geometric median runs at --rule-scope model, where both parameter
# servers take the same Weiszfeld weights
RULES = {"mean": dict(mode="normal"), "median": dict(mode="coordinate_median"), "multi_krum": dict(mode="multi_krum"),
         "bulyan": dict(mode="bulyan", num_workers=7, worker_fail=1),
         "geomedian": dict(mode="geometric_median", rule_scope="model"),
         "centered_clip": dict(mode="centered_clip", clip_tau=0.5),
         "detox_median": dict(approach="detox", mode="coordinate_median", num_workers=9, group_size=3),
         "nnm_median": dict(approach="nnm", mode="coordinate_median"),
         "bucketed_median": dict(mode="coordinate_median", bucketing=2)}


@pytest.mark.parametrize("scope", ["tensor", "model"])
@pytest.mark.parametrize("rule", list(RULES))
def test_fused_arc_matches_the_library_op_engine(monkeypatch, rule, scope):
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    kw = dict(RULES[rule], arc=scope)
    a, _ = _run(_cfg(**kw), 4)
    b, _ = _run(_cfg(transport="nccl", **kw), 4)
    assert a.engine.ps.arc_ws is not None and (scope == "tensor" or not a.engine.pipeline_ps)
    assert (a.engine.ps.arc_ws.factors < 1).any()
    pa, pb = a.engine.master_params(), b.engine.master_params()
    assert torch.isfinite(pa).all()
    assert torch.allclose(pa, pb, atol=2e-5), float((pa - pb).abs().max())


_RESNET = dict(network="ResNet18", dataset="Cifar10", batch_size=8, dtype="bf16", synthetic_size=256, err_mode="alie",
               num_workers=7, worker_fail=1, mode="coordinate_median")


@pytest.mark.parametrize("scope", ["tensor", "model"])
def test_graph_replay_equals_eager(scope):
    e, le = _run(_cfg(cuda_graphs=False, arc=scope, **_RESNET), 5)
    g, lg = _run(_cfg(cuda_graphs=True, arc=scope, **_RESNET), 5)
    assert g.engine.graph is not None and g.engine.pipeline_ps == (scope == "tensor")
    assert torch.equal(e.engine.master_params(), g.engine.master_params())
    assert le == lg and all(np.isfinite(lg))


@pytest.mark.parametrize("scope", ["tensor", "model"])
def test_f_zero_is_bit_identical_to_no_arc(scope):
    kw = dict(_RESNET, worker_fail=0, err_mode="none", cuda_graphs=True)
    a, la = _run(_cfg(arc=scope, **kw), 5)
    b, lb = _run(_cfg(**kw), 5)
    assert a.engine.ps.arc_ws is None and a.engine.pipeline_ps == b.engine.pipeline_ps
    assert a.engine.kernels_per_step == b.engine.kernels_per_step
    assert torch.equal(a.engine.master_params(), b.engine.master_params()) and la == lb


def test_debug_checksum_skips_the_rescaled_slots():
    t, _ = _run(_cfg(mode="coordinate_median", err_mode="alie", worker_fail=2, arc="model", debug_checksum=True), 3)
    log = t.engine.checksum_log
    assert len(log) == 3 and all(r["bad"] == [] for r in log), log
    # ALIE overwrites the two liar slots; ARC rescales k = 2 slots, which may include liars
    assert all(7 - 2 - oracle.arc_k(7, 2) <= r["checked"] <= 7 - 2 for r in log), log
    rescaled = (t.engine.ps.arc_ws.factors < 1).any(0).cpu()
    assert int(rescaled.sum()) == oracle.arc_k(7, 2)


@pytest.mark.parametrize("scope", ["tensor", "model"])
def test_debug_checksum_and_compression_compose(scope):
    a, la = _run(_cfg(mode="coordinate_median", arc=scope, debug_checksum=True), 3)
    b, lb = _run(_cfg(mode="coordinate_median", arc=scope, compress_grad="compress"), 3)
    c, lc = _run(_cfg(mode="coordinate_median", arc=scope), 3)
    assert all(r["bad"] == [] for r in a.engine.checksum_log)
    assert torch.equal(a.engine.master_params(), c.engine.master_params())
    assert torch.equal(b.engine.master_params(), c.engine.master_params())
    assert la == lb == lc


def test_the_mean_with_arc_trains_under_sign_flip_liars_where_the_plain_mean_does_not():
    """The clipped liars still pull against the honest rows, so the mean with ARC trains more slowly than the clean job."""
    kw = dict(mode="normal", num_workers=7, worker_fail=2, err_mode="rev_grad", lr=0.05, max_steps=18)
    clean, lc = _run(_cfg(err_mode="none", **{k: v for k, v in kw.items() if k != "err_mode"}), 16)
    arc, la = _run(_cfg(arc="tensor", **kw), 16)
    mean, lm = _run(_cfg(**kw), 16)
    assert np.isfinite(la).all() and la[-1] < la[0], (la, lc, lm)
    pc = clean.engine.master_params()
    d_arc = float((arc.engine.master_params() - pc).norm())
    d_mean = float((mean.engine.master_params() - pc).norm())
    assert not d_mean < 10 * d_arc, (d_arc, d_mean)              # the mean leaves the clean trajectory (or turns NaN)
