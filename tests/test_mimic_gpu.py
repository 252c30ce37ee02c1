"""The mimic and IPM attacks on the GPU (csrc/cuda/mimic.cu, attack_ipm_kernel in csrc/cuda/attack.cu): the kernels against the
fp64 oracle of codes/adversary.py on the ResNet-18 arena, their invariance to the grid size and the gradient-bucket cuts, a 2W-step
chain against the oracle, and whole fused jobs (captured graph against eager, nvl against nccl, resume inside the warm-up, the
defences that compose with the attacks, the transport self-check)."""
import numpy as np
import pytest
import torch

from draco_b200 import JobConfig
from draco_b200.codes import adversary as A
from draco_b200.models import build_model
from draco_b200.parallel.arena import ArenaLayout
from draco_b200.parallel.trainer import Trainer

pytestmark = pytest.mark.gpu
INF, NAN = float("inf"), float("nan")


@pytest.fixture(scope="module")
def K():
    from draco_b200.ops import kernels
    return kernels


@pytest.fixture(scope="module")
def L():
    return ArenaLayout.from_model(build_model("ResNet18"), bf16=True, channels_last=True)


@pytest.fixture(scope="module")
def spans(L):
    return [(s.offset, s.numel) for s in L.specs]


@pytest.fixture(scope="module")
def z0(L, spans):
    return A.mimic_z0(spans, L.total)


def slab(L, P, seed, special=True, z=None, spread=0.0):
    """[P, D] fp32 on the host: N(0, 1) rows scaled per tensor, padding zero.  With ``special``, worker 0 holds +Inf in tensor 3,
    -Inf in tensor 5, 1e30 in tensor 7 and NaN in tensor 9 (one coordinate each).  ``spread``: row i moves by i * spread * z, so
    the projections on z lie that far apart."""
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((P, L.total)).astype(np.float32)
    for t, s in enumerate(L.specs):
        X[:, s.offset:s.offset + s.numel] *= np.float32(10.0 ** ((t % 5) - 2))
    if spread:
        order = rng.permutation(P)
        X += (order[:, None] * spread * z[None, :]).astype(np.float32)
    X[:, ~L.valid_mask()] = 0
    if special:
        for t, v in ((3, INF), (5, -INF), (7, 1e30), (9, NAN)):
            X[0, L.specs[t].offset + 1] = v
    return X


def bitmap(liars_per_step):
    out = []
    for liars in liars_per_step:
        bm = 0
        for w in liars:
            bm |= 1 << w
        out.append(bm)
    return torch.tensor(out, dtype=torch.int32, device="cuda")


def same_bits(a, b):
    """Bit-equal, except that any NaN equals any NaN (the device's NaN payload is not numpy's)."""
    a, b = np.asarray(a, dtype=np.float32), np.asarray(b, dtype=np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.int32), b[~nb].view(np.int32))


def _liars(P, rng):
    """f = 1, P - 1 or in between; worker 0 (the one holding the special values) is honest."""
    f = [1, P - 1, int(rng.integers(1, P))][P % 3]
    return sorted((1 + rng.choice(P - 1, size=f, replace=False)).tolist())


def mimic_dev(K, L, X, liars_per_step, z0, W, steps, grid=None):
    """``steps`` device steps of the mimic chain from m = 0 and z = ``z0``; X is one slab, or one per step."""
    P = X[0].shape[0] if isinstance(X, list) else X.shape[0]
    st = K.MimicState(L, P, torch.device("cuda"), torch.from_numpy(z0))
    n = len(liars_per_step)
    bm = bitmap([liars_per_step[(i - 1) % n] for i in range(n)])     # step s reads entry s % n: liars_per_step[s - 1]
    out, targets = [], []
    for step in range(1, steps + 1):
        g = torch.from_numpy(X[step - 1] if isinstance(X, list) else X).cuda().contiguous()
        K.mimic_step(L, g, L.total, P, adv_bitmap=bm, adv_len=len(liars_per_step),
                     step_ptr=torch.full((1,), step, dtype=torch.int64, device="cuda"), warmup=W, st=st, grid=grid)
        torch.cuda.synchronize()
        out.append(g.cpu().numpy())
        targets.append(int(st.target.item()))
    return out, targets, st


# z after a warm-up step: the device folds the whole-model sums s_i, <m', z> and ||u||^2 tile by tile (fma, warp shuffles)
# instead of numpy's pairwise order.  Each is a sum of at most D = 1.1e7 terms, so its error is at most D 2^-53 sum|terms|, about
# 1.2e-9 relative to the sum of magnitudes.  On these slabs sum|x_i z| is ~1e5 and the s_i lie ~1e3 apart, so w_i moves by < 1e-7 relative, u
# (linear in the w_i) by < 1e-7 relative to ||u||, and z = u / ||u|| by < 2e-7 in norm, plus fp32 rounding (<= 2^-24 per
# element, ||.|| <= 6e-8): ||z_gpu - z_ref|| <= 1e-6.  m' has the same operations on both sides: bit for bit.
Z_TOL = 1e-6


@pytest.mark.parametrize("P", range(3, 17))
def test_mimic_kernels_match_the_fp64_oracle(K, L, spans, z0, P):
    rng = np.random.default_rng(P)
    liars = _liars(P, rng)
    honest = [w for w in range(P) if w not in liars]
    pad = ~L.valid_mask()
    # (a) the special-value slab: worker 0's NaN makes s_0 NaN, the largest, so every liar copies worker 0; u and z turn NaN
    X = slab(L, P, seed=P)
    (got,), (k,), st = mimic_dev(K, L, X, [liars], z0, W=1, steps=1)
    ref, kr, sr = A.mimic_step(X, liars, spans, A.MimicState(np.zeros(L.total, np.float32), z0), t=0, W=1)
    assert k == kr == 0
    assert same_bits(got[honest], X[honest]) and same_bits(got[:, pad], X[:, pad])
    for w in liars:
        assert np.array_equal(got[w][~pad].view(np.int32), X[0][~pad].view(np.int32))
    assert same_bits(st.m.cpu().numpy(), sr.m)
    assert np.isnan(sr.z[~pad]).all() and np.isnan(st.z.cpu().numpy()[~pad]).all()
    # (b) finite rows whose projections lie ~1000 apart: the device's target is the oracle's, and the state after the update
    X = slab(L, P, seed=100 + P, special=False, z=z0, spread=1000.0)
    (got,), (k,), st = mimic_dev(K, L, X, [liars], z0, W=1, steps=1)
    ref, kr, sr = A.mimic_step(X, liars, spans, A.MimicState(np.zeros(L.total, np.float32), z0), t=0, W=1)
    s = sorted(float(X[i].astype(np.float64) @ z0.astype(np.float64)) for i in honest)
    assert len(s) < 2 or s[-1] - s[-2] > 100.0
    assert k == kr
    assert same_bits(got, ref)
    assert same_bits(st.m.cpu().numpy(), sr.m)
    zg = st.z.cpu().numpy()
    assert np.all(zg[pad] == 0)
    assert float(np.linalg.norm(zg.astype(np.float64) - sr.z.astype(np.float64))) <= Z_TOL


def test_mimic_is_independent_of_the_grid_and_returns_after_the_warm_up(K, L, z0):
    P = 9
    X = [slab(L, P, seed=s, special=False, z=z0, spread=1000.0) for s in range(4)]
    liars = [[1, 4], [2, 3, 7], [0, 8], [5]]
    ref, tref, sref = mimic_dev(K, L, X, liars, z0, W=2, steps=4)
    for grid in (1, 37):
        got, t, st = mimic_dev(K, L, X, liars, z0, W=2, steps=4, grid=grid)
        assert t == tref and all(np.array_equal(a.view(np.int32), b.view(np.int32)) for a, b in zip(got, ref))
        assert torch.equal(st.m, sref.m) and torch.equal(st.z, sref.z)
    # past W the state is frozen: steps 3 and 4 (t = 2, 3) leave m and z as step 2 left them
    _, _, s2 = mimic_dev(K, L, X, liars, z0, W=2, steps=2)
    assert torch.equal(s2.m, sref.m) and torch.equal(s2.z, sref.z)


def test_2w_steps_of_the_chain_follow_the_oracle(K, L, spans, z0):
    """W = 3, six steps with a new slab and liar set each step: the same target sequence, m bit for bit, and z within Z_TOL per
    step (the errors do not compound: each update renormalises)."""
    P, W = 7, 3
    rng = np.random.default_rng(11)
    X = [slab(L, P, seed=50 + t, special=False, z=z0, spread=1000.0) for t in range(2 * W)]
    liars = [sorted(rng.choice(P, size=2, replace=False).tolist()) for _ in range(2 * W)]
    got, tg, st = mimic_dev(K, L, X, liars, z0, W=W, steps=2 * W)
    s = A.MimicState(np.zeros(L.total, np.float32), z0)
    tr = []
    for t in range(2 * W):
        ref, k, s = A.mimic_step(X[t], liars[t], spans, s, t=t, W=W)
        tr.append(k)
        assert same_bits(got[t], ref), t
    assert tg == tr
    assert same_bits(st.m.cpu().numpy(), s.m)
    assert float(np.linalg.norm(st.z.cpu().numpy().astype(np.float64) - s.z.astype(np.float64))) <= 2 * W * Z_TOL


@pytest.mark.parametrize("P", range(3, 17))
def test_ipm_kernel_matches_the_fp64_oracle_per_bucket(K, L, spans, P):
    """The kernel forms the oracle's fp64 mean with the same operations (sum from +0 in slot order, one division) and one
    rounded product: the row is the oracle's fp64 row rounded to fp32, bit for bit (NaN where it is NaN)."""
    rng = np.random.default_rng(P)
    X = slab(L, P, seed=P)
    liars = _liars(P, rng)
    honest = [w for w in range(P) if w not in liars]
    eps = 0.1 * (1 + P % 3)
    ref = A.ps_attack(X, liars, "ipm", spans, z=eps)
    g = torch.from_numpy(X).cuda().contiguous()
    # three gradient buckets of whole tensors, like the pipelined PS's
    cuts = [0, L.ntensors // 3, 2 * L.ntensors // 3, L.ntensors]
    for b in range(3):
        t0, t1 = cuts[b], cuts[b + 1]
        tiles = (L.specs[t0].offset // 1024, (L.specs[t1 - 1].offset + L.specs[t1 - 1].numel + 1023) // 1024)
        n = K.ps_attack(L, g, L.total, P, A.ATTACK_IPM, adv_bitmap=bitmap([liars]), adv_len=1,
                        step_ptr=torch.ones(1, dtype=torch.int64, device="cuda"), z=eps, tile_range=tiles, tensor_range=(t0, t1))
        assert n == 1
    torch.cuda.synchronize()
    got = g.cpu().numpy()
    assert same_bits(got, ref)
    assert same_bits(got[honest], X[honest])
    for grid in (None, 1, 37):
        h = torch.from_numpy(X).cuda().contiguous()
        K.ps_attack(L, h, L.total, P, A.ATTACK_IPM, adv_bitmap=bitmap([liars]), adv_len=1,
                    step_ptr=torch.ones(1, dtype=torch.int64, device="cuda"), z=eps, grid=grid)
        torch.cuda.synchronize()
        assert same_bits(h.cpu().numpy(), got), grid


# ------------------------------------------------------------------------------------------------ engine
def _cfg(**kw):
    base = dict(network="LeNet", dataset="MNIST", batch_size=16, max_steps=12, num_workers=7, transport="nvl", lr=0.02,
                momentum=0.9, synthetic_size=512, eval_freq=10 ** 6, compress_grad="None", dtype="fp32", cuda_graphs=False,
                approach="baseline", mode="coordinate_median", worker_fail=2)
    base.update(kw)
    return JobConfig(**base)


def _run(cfg, steps):
    t = Trainer(cfg, rank=0, world=1, device=torch.device("cuda", 0), quiet=True)
    losses = [t.train_step()["loss"] for _ in range(steps)]
    t.synchronize()
    return t, losses


_RESNET = dict(network="ResNet18", dataset="Cifar10", batch_size=8, dtype="bf16", synthetic_size=256, approach="baseline",
               mode="trimmed_mean", num_workers=7, worker_fail=2)


@pytest.mark.parametrize("mode", ["ipm", "mimic"])
def test_attack_runs_inside_the_captured_graph_and_replay_equals_eager(mode):
    kw = dict(err_mode=mode, mimic_warmup=4 if mode == "mimic" else None, **_RESNET)
    e, le = _run(_cfg(cuda_graphs=False, **kw), 7)
    g, lg = _run(_cfg(cuda_graphs=True, **kw), 7)
    eng = g.engine
    assert eng.graph is not None and eng.ps.attack == A.attack_code(mode)
    assert eng.pipeline_ps == (mode == "ipm")                       # mimic leaves the pipelined PS
    assert torch.equal(e.engine.master_params(), eng.master_params())
    assert le == lg
    if mode == "mimic":
        assert torch.equal(e.engine.ps.mimic.z, eng.ps.mimic.z) and torch.equal(e.engine.ps.mimic.m, eng.ps.mimic.m)
    clean, _ = _run(_cfg(cuda_graphs=True, err_mode="none", **_RESNET), 7)
    assert not torch.equal(clean.engine.master_params(), eng.master_params())


@pytest.mark.parametrize("mode", ["ipm", "mimic"])
def test_fused_attack_matches_library_op_engine(monkeypatch, mode):
    """Mimic: the same targets as long as the projections are not within rounding of each other, so the same slots, and the same
    m; z differs by rounding.  IPM: rows bit for bit.  4 LeNet steps at lr 0.02 keep the parameters within 1e-4."""
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    kw = dict(err_mode=mode, mimic_warmup=2 if mode == "mimic" else None)
    a, _ = _run(_cfg(**kw), 4)
    b, _ = _run(_cfg(transport="nccl", **kw), 4)
    pa, pb = a.engine.master_params(), b.engine.master_params()
    assert torch.isfinite(pa).all()
    assert torch.allclose(pa, pb, atol=1e-4), float((pa - pb).abs().max())
    if mode == "mimic":
        za, zb = a.engine.ps.mimic.z, b.engine.ps.mimic_z
        assert float((za.double() - zb.double()).norm()) <= 1e-4


def test_resume_inside_the_warm_up_is_bit_for_bit(tmp_path):
    d = str(tmp_path) + "/"
    kw = dict(err_mode="mimic", mimic_warmup=5, train_dir=d, max_steps=8, cuda_graphs=True)
    t = Trainer(_cfg(eval_freq=3, **kw), rank=0, world=1, device=torch.device("cuda", 0), quiet=True)
    t.fit(8)
    t.synchronize()
    final, m, z = t.engine.master_params().clone(), t.engine.ps.mimic.m.clone(), t.engine.ps.mimic.z.clone()
    t.close()
    t2 = Trainer(_cfg(eval_freq=10 ** 6, checkpoint_step=3, **kw), rank=0, world=1, device=torch.device("cuda", 0), quiet=True)
    assert t2.step == 4
    for _ in range(5):
        t2.train_step()
    t2.synchronize()
    assert torch.equal(t2.engine.master_params(), final)
    assert torch.equal(t2.engine.ps.mimic.m, m) and torch.equal(t2.engine.ps.mimic.z, z)


@pytest.mark.parametrize("mode", ["ipm", "mimic"])
@pytest.mark.parametrize("extra", [dict(bucketing=2, worker_fail=1), dict(worker_momentum=0.9, momentum=0.0),
                                   dict(approach="detox", group_size=3, num_workers=9),
                                   dict(approach="nnm", mode="coordinate_median")])
def test_the_defences_run_finite_under_the_attack(mode, extra):
    kw = dict(dict(_RESNET, mode="coordinate_median", cuda_graphs=True, err_mode=mode,
                   mimic_warmup=3 if mode == "mimic" else None), **extra)
    t, losses = _run(_cfg(**kw), 6)
    assert t.engine.graph is not None
    assert all(np.isfinite(losses)) and torch.isfinite(t.engine.master_params()).all()


@pytest.mark.parametrize("mode", ["ipm", "mimic"])
def test_debug_checksum_skips_the_overwritten_liar_slots(mode):
    t, _ = _run(_cfg(err_mode=mode, debug_checksum=True), 3)
    log = t.engine.checksum_log
    assert len(log) == 3 and all(r["bad"] == [] and r["checked"] == 7 - 2 for r in log), log
