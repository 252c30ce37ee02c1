"""The ALIE and min-max attacks on the GPU (csrc/cuda/attack.cu): the PS-side kernels against the fp64 oracle of
codes/adversary.py on the ResNet-18 arena layout, their invariance to the grid size and the bucketing, and whole fused-engine
jobs under each attack (captured graph, pipelined PS and worker streams kept; replay == eager; exact recovery by the vote;
the library-op engine; the compressed wire; the transport self-check)."""
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
EPS64, EPS32 = 2.0 ** -53, 2.0 ** -24


@pytest.fixture(scope="module")
def K():
    from draco_b200.ops import kernels
    return kernels


@pytest.fixture(scope="module")
def L():
    return ArenaLayout.from_model(build_model("ResNet18"), bf16=True, channels_last=True)


def slab(L, P, seed, special=True):
    """[P, D] fp32 on the host: N(0, 1) rows scaled per tensor, padding zero.  With ``special``, worker 0 holds +Inf in tensor 3,
    -Inf in tensor 5, 1e30 in tensor 7 and NaN in tensor 9 (one coordinate each)."""
    rng = np.random.default_rng(seed)
    X = rng.standard_normal((P, L.total)).astype(np.float32)
    for t, s in enumerate(L.specs):
        X[:, s.offset:s.offset + s.numel] *= np.float32(10.0 ** ((t % 5) - 2))
    X[:, ~L.valid_mask()] = 0
    if special:
        for t, v in ((3, INF), (5, -INF), (7, 1e30), (9, NAN)):
            X[0, L.specs[t].offset + 1] = v
    return X


def bitmap(P, liars):
    bm = 0
    for w in liars:
        bm |= 1 << w
    return torch.tensor([bm], dtype=torch.int32, device="cuda")


def run(K, L, X, liars, mode, z=0.0, **kw):
    P = X.shape[0]
    g = torch.from_numpy(X).cuda().contiguous()
    ws = K.AttackWorkspace(L, P, g.device) if mode == "minmax" else None
    K.ps_attack(L, g, L.total, P, A.attack_code(mode), adv_bitmap=bitmap(P, liars), adv_len=1,
                step_ptr=torch.ones(1, dtype=torch.int64, device="cuda"), z=z, ws=ws, **kw)
    torch.cuda.synchronize()
    return g, ws


def same_bits(a, b):
    return np.array_equal(np.asarray(a).view(np.int32), np.asarray(b).view(np.int32))


def _liars(P, rng):
    """f = 1, P - 1 or in between; worker 0 (the one holding the special values) is honest."""
    f = [1, P - 1, int(rng.integers(1, P))][P % 3]
    return sorted((1 + rng.choice(P - 1, size=f, replace=False)).tolist())


@pytest.mark.parametrize("mode", ["alie", "minmax"])
@pytest.mark.parametrize("P", range(3, 17))
def test_attack_kernels_match_the_fp64_oracle(K, L, P, mode):
    """Per element, with M = max_i |g_i| over the honest rows, n = n_h, mu / sigma / gamma the oracle's:

    * both sides form mu and sigma with n + 2 fp64 roundings each and the row with 2 more, so their fp64 rows differ by at most
      e64 = (2 n + 8) 2^-53 M (1 + z) (ALIE; min-max with gamma for z); the kernel follows the oracle's operation order, so in
      practice this is 0;
    * ALIE: each side rounds to fp32 once: |got - ref| <= 2^-24 (|got| + |ref|) + e64;
    * min-max: the write pass reads mu and sigma rounded to fp32 (2^-24 |mu|, 2^-24 gamma sigma) and a gamma whose per-tensor
      fp64 sums are folded tile by tile instead of numpy's order.  For the sums of non-negative terms (a_i, c, Dmax^2) that moves
      each by at most D eps64 relative, D < 2.4e6 elements per tensor: 3e-10.  b_i is a signed sum, but it enters gamma next to
      c (Dmax^2 - a_i), which dominates on these rows; the test allows |gamma_k - gamma| <= 1e-8 gamma (checked on its own), so
      |got - ref| <= 2^-24 (|mu| + gamma sigma + |got| + |ref|) + 1e-8 gamma sigma + e64.
    Where the oracle's row is not finite the kernel's is the same value (NaN where it is NaN)."""
    rng = np.random.default_rng(P)
    X = slab(L, P, seed=P)
    liars = _liars(P, rng)
    honest = [w for w in range(P) if w not in liars]
    z = A.alie_z_max(P, len(liars)) if A.alie_s(P, len(liars)) >= 1 else 1.5
    g, ws = run(K, L, X, liars, mode, z)
    got = g.cpu().numpy()
    assert same_bits(got[honest], X[honest])                                    # honest slots untouched
    pad = ~L.valid_mask()
    assert same_bits(got[:, pad], X[:, pad])                                    # padding untouched
    for w in liars[1:]:
        assert same_bits(got[w], got[liars[0]])                                 # every liar sends the same row
    row = got[liars[0]]
    n = len(honest)
    for t, s in enumerate(L.specs):
        H = X[honest, s.offset:s.offset + s.numel].astype(np.float64)
        mu, sd = A.honest_stats(H)
        k = z
        if mode == "alie":
            ref64 = A.alie_row(H, z)
        else:
            gam = A.minmax_gamma(H)
            gk = float(ws.gamma[t])
            if np.isnan(gam):
                assert np.isnan(gk), t
            else:
                assert abs(gk - gam) <= 1e-8 * gam, (t, gk, gam)
            k = gam
            ref64 = A.minmax_row(H)
        with np.errstate(over="ignore", invalid="ignore"):
            ref = ref64.astype(np.float32).astype(np.float64)
            r = row[s.offset:s.offset + s.numel].astype(np.float64)
            M = np.abs(H).max(0)
            e64 = (2 * n + 8) * EPS64 * M * (1 + abs(k))
            bound = EPS32 * (np.abs(r) + np.abs(ref)) + e64
            if mode == "minmax":
                bound = bound + EPS32 * (np.abs(mu) + k * sd) + 1e-8 * k * sd
            fin = np.isfinite(ref)
            assert np.all(np.abs(r[fin] - ref[fin]) <= bound[fin]), (t, float(np.nanmax(np.abs(r[fin] - ref[fin]) - bound[fin])))
            nf = ~fin
            assert np.array_equal(np.isnan(r[nf]), np.isnan(ref[nf])), t
            assert np.array_equal(r[nf][~np.isnan(ref[nf])], ref[nf][~np.isnan(ref[nf])]), t
    if mode == "minmax":                                                         # the tensors that hold +-Inf / NaN: NaN gamma
        assert np.isnan(row[L.specs[3].offset]) and np.isnan(row[L.specs[9].offset])
        assert np.isfinite(row[L.specs[7].offset:L.specs[7].offset + L.specs[7].numel]).all()


@pytest.mark.parametrize("mode", ["alie", "minmax"])
def test_attack_is_independent_of_grid_and_buckets(K, L, mode):
    P, liars = 15, [2, 7, 11]
    X = slab(L, P, seed=5, special=False)
    z = A.alie_z_max(P, 3)
    ref, _ = run(K, L, X, liars, mode, z)
    # buckets of whole tensors, as the pipelined PS cuts the arena
    cuts = [0, 10, 11, 40, L.ntensors]
    tile0 = [L.specs[i].offset // 1024 for i in cuts[:-1]] + [L.ntiles]
    g = torch.from_numpy(X).cuda().contiguous()
    ws = K.AttackWorkspace(L, P, g.device) if mode == "minmax" else None
    step = torch.ones(1, dtype=torch.int64, device="cuda")
    for b in range(len(cuts) - 1):
        K.ps_attack(L, g, L.total, P, A.attack_code(mode), adv_bitmap=bitmap(P, liars), adv_len=1, step_ptr=step, z=z, ws=ws,
                    tile_range=(tile0[b], tile0[b + 1]), tensor_range=(cuts[b], cuts[b + 1]))
    torch.cuda.synchronize()
    assert torch.equal(g, ref)
    for grid in (1, 37):
        h, _ = run(K, L, X, liars, mode, z, grid=grid)
        assert torch.equal(h, ref), grid
    assert not torch.equal(ref, torch.from_numpy(X).cuda())


def test_attack_reads_the_liar_set_of_the_device_step(K, L):
    """The liar set is adv_bitmap[step % adv_len]: an empty bitmap leaves the slab alone, the step picks the entry."""
    P = 5
    X = slab(L, P, seed=9, special=False)
    g = torch.from_numpy(X).cuda().contiguous()
    bm = torch.tensor([0b00100, 0, 0b00011], dtype=torch.int32, device="cuda")
    for step, liars in ((4, []), (5, [0, 1]), (3, [2])):
        h = g.clone()
        K.ps_attack(L, h, L.total, P, 5, adv_bitmap=bm, adv_len=3, step_ptr=torch.full((1,), step, dtype=torch.int64, device="cuda"),
                    z=1.0)
        torch.cuda.synchronize()
        changed = [w for w in range(P) if not torch.equal(h[w], g[w])]
        assert changed == liars, (step, changed)


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


@pytest.mark.parametrize("mode", ["alie", "minmax"])
def test_attack_runs_inside_the_captured_graph_and_replay_equals_eager(mode):
    e, le = _run(_cfg(cuda_graphs=False, err_mode=mode, **_RESNET), 6)
    g, lg = _run(_cfg(cuda_graphs=True, err_mode=mode, **_RESNET), 6)
    eng = g.engine
    assert eng.graph is not None and eng.pipeline_ps and len(eng.worker_streams) > 1 and eng.ps.attack == A.attack_code(mode)
    assert torch.equal(e.engine.master_params(), eng.master_params())
    assert le == lg
    clean, _ = _run(_cfg(cuda_graphs=True, err_mode="none", **_RESNET), 6)
    assert not torch.equal(clean.engine.master_params(), eng.master_params())     # the attack reached the update


@pytest.mark.parametrize("mode", ["alie", "minmax"])
def test_vote_recovers_exactly_while_no_group_is_captured(mode):
    """Groups of 3 and one liar per step: every group keeps an honest majority, so the vote returns the honest gradient and
    the run is bit-identical to the attack-free one (graph mode, pipelined PS, worker streams)."""
    kw = dict(_RESNET, approach="maj_vote", mode="maj_vote", num_workers=6, group_size=3, worker_fail=1, cuda_graphs=True)
    clean, lc = _run(_cfg(err_mode="none", **kw), 6)
    att, la = _run(_cfg(err_mode=mode, **kw), 6)
    assert att.engine.graph is not None and att.engine.pipeline_ps
    assert torch.equal(clean.engine.master_params(), att.engine.master_params())
    assert lc == la


@pytest.mark.parametrize("err_mode", ["alie", "minmax"])
@pytest.mark.parametrize("rule", [dict(mode="coordinate_median"), dict(mode="multi_krum", num_workers=9),
                                  dict(approach="detox", mode="trimmed_mean", num_workers=9, group_size=3)])
def test_fused_attack_matches_library_op_engine(monkeypatch, err_mode, rule):
    """Same rows up to the fp32 rounding of mu and sigma in the min-max write pass (a few ulps); 4 LeNet steps at lr 0.02 keep
    the parameters within 1e-4."""
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    kw = dict(err_mode=err_mode, **rule)
    a, _ = _run(_cfg(**kw), 4)
    b, _ = _run(_cfg(transport="nccl", **kw), 4)
    pa, pb = a.engine.master_params(), b.engine.master_params()
    assert torch.isfinite(pa).all()
    assert torch.allclose(pa, pb, atol=1e-4), float((pa - pb).abs().max())


@pytest.mark.parametrize("mode", ["alie", "minmax"])
def test_compressed_wire_gives_the_same_bits(mode):
    a, la = _run(_cfg(err_mode=mode), 4)
    b, lb = _run(_cfg(err_mode=mode, compress_grad="compress"), 4)
    assert a.engine.pipeline_ps and not b.engine.pipeline_ps
    assert torch.equal(a.engine.master_params(), b.engine.master_params())
    assert la == lb


@pytest.mark.parametrize("mode", ["alie", "minmax"])
def test_debug_checksum_skips_the_overwritten_liar_slots(mode):
    t, _ = _run(_cfg(err_mode=mode, debug_checksum=True), 3)
    log = t.engine.checksum_log
    assert len(log) == 3 and all(r["bad"] == [] and r["checked"] == 7 - 2 for r in log), log
