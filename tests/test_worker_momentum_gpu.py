"""Worker-side momentum on the GPU: the momentum build of the push kernel (csrc/cuda/push_encode.cu) bit for bit against an fp32
torch restatement of ``codes/oracle.py worker_momentum`` in both gradient modes, bucketing, the adversary hook, padding, and the
argument checks; then whole jobs on the fused engine against the library-op engine, under graph replay, worker streams, the
compressed wire, --debug-checksum, the PS-side attacks, the vote, and resume."""
import numpy as np
import pytest
import torch

from draco_b200 import JobConfig
from draco_b200.codes import adversary as A
from draco_b200.codes import oracle
from draco_b200.models import build_model
from draco_b200.parallel.arena import ArenaLayout
from draco_b200.parallel.trainer import Trainer
from draco_b200.utils.checkpoint import load_checkpoint

pytestmark = pytest.mark.gpu
BETA = 0.9


@pytest.fixture(scope="module")
def K():
    from draco_b200.ops import kernels
    return kernels


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def L():
    # ResNet-18 in bf16: bf16 convolution / linear tensors and fp32 BatchNorm tensors, every tensor padded to a tile
    return ArenaLayout.from_model(build_model("ResNet18"), bf16=True, channels_last=True)


def _grads(L, dev, seed):
    """One step's gradient: fp32 arena + bf16 arena (each tensor in its own dtype, padding zero), per-tensor copies for the
    zero-copy table (padding-free, in arena element order), and the widened fp32 flat gradient."""
    g = torch.Generator().manual_seed(seed)
    g32 = L.new_arena(dev)
    g16 = L.new_arena(dev, torch.bfloat16)
    per = []
    for s in L.specs:
        v = (torch.randn(s.numel, generator=g) * 0.1).to(dev)
        if s.is_bf16:
            v = v.to(torch.bfloat16)
            g16[s.offset: s.offset + s.numel] = v
        else:
            g32[s.offset: s.offset + s.numel] = v
        per.append(v.clone())
    flat = g32.clone()
    for s, v in zip(L.specs, per):
        flat[s.offset: s.offset + s.numel] = v.float()
    table = torch.tensor([[v.data_ptr() for v in per]], dtype=torch.int64, device=dev)
    return g32, g16, per, table, flat


def _restate(m, g):
    b, c = oracle.worker_momentum_coefficients(BETA)
    m.mul_(b)
    m.add_(g * c)


class _Push:
    def __init__(self, K, L, dev, attack=0):
        self.K, self.L = K, L
        self.step = torch.ones(1, dtype=torch.int64, device=dev)
        self.cnt = torch.zeros(1, dtype=torch.int32, device=dev)
        self.bitmap = torch.tensor([1 << 2], dtype=torch.int32, device=dev)      # worker slot 2 lies every step
        self.attack = attack

    def __call__(self, g32, g16, dst, wmom, table=None, tile_range=None, grid=None, local_copy=None):
        self.K.push_encode(self.L, [g32], [g16], dst, step_ptr=self.step, worker=2, done_counter=self.cnt,
                           adv_bitmap=self.bitmap if self.attack else None, adv_len=1 if self.attack else 0, attack=self.attack,
                           magnitude=-100.0, seed=5, src_table=table, tile_range=tile_range, grid=grid, local_copy=local_copy,
                           wmom=wmom, wm_beta=BETA)


@pytest.mark.parametrize("zero_copy", [False, True])
@pytest.mark.parametrize("attack", [0, 1, 2, 3])
def test_momentum_push_matches_the_torch_restatement(K, L, dev, zero_copy, attack):
    valid = torch.from_numpy(L.valid_mask()).to(dev)
    push = _Push(K, L, dev, attack)
    wm = L.new_arena(dev)
    m_ref = L.new_arena(dev)
    slot = L.new_arena(dev)                                        # slots and copies start zeroed, as the engine's do
    copy = torch.full((L.total,), 7.0, device=dev)
    copy[~valid] = 0
    for step in range(1, 4):
        push.step.fill_(step)
        g32, g16, _, table, flat = _grads(L, dev, seed=10 * step + zero_copy)
        push(g32, g16, slot, wm, table=table if zero_copy else None, local_copy=copy)
        torch.cuda.synchronize()
        _restate(m_ref, flat)
        assert torch.equal(wm, m_ref), step                        # the state follows the true gradient, liar or not
        if attack == 0:
            want = m_ref
        elif attack == 1:
            want = m_ref * -100.0
        elif attack == 2:
            want = torch.where(valid, torch.full_like(m_ref, -100.0), torch.zeros_like(m_ref))
        if attack in (0, 1, 2):
            assert torch.equal(slot[valid], want[valid]), step
        else:                                                      # random: a fresh normal row, nothing of the state in it
            assert not torch.equal(slot[valid], m_ref[valid]) and torch.isfinite(slot).all()
        assert torch.equal(copy, slot)
        assert float(wm[~valid].abs().sum()) == 0 and float(slot[~valid].abs().sum()) == 0
        assert int(wm[~valid].view(torch.int32).abs().sum()) == 0     # +0 padding, not -0
    assert push.cnt.item() == 0


def test_bucketed_pushes_equal_one_whole_push(K, L, dev):
    nt = L.ntiles
    bounds = [0, nt // 7, nt // 7 + 1, nt // 2, nt - 3, nt]
    out = []
    for how in ("whole", "buckets", "grid5"):
        push = _Push(K, L, dev, attack=1)
        wm = L.new_arena(dev)
        slot = L.new_arena(dev)
        for step in range(1, 4):
            push.step.fill_(step)
            g32, g16, _, table, _ = _grads(L, dev, seed=step)
            if how == "buckets":
                for i in range(len(bounds) - 1):
                    push(g32, g16, slot, wm, table=table, tile_range=(bounds[i], bounds[i + 1]), grid=3)
            else:
                push(g32, g16, slot, wm, table=table, grid=5 if how == "grid5" else None)
        torch.cuda.synchronize()
        out.append((wm, slot))
    for wm, slot in out[1:]:
        assert torch.equal(wm, out[0][0]) and torch.equal(slot, out[0][1])


def test_plain_push_is_unchanged_and_the_launcher_checks_arguments(K, L, dev):
    push = _Push(K, L, dev)
    g32, g16, _, table, flat = _grads(L, dev, seed=3)
    slot = L.new_arena(dev)
    K.push_encode(L, [g32], [g16], slot, step_ptr=push.step, worker=2, done_counter=push.cnt)
    torch.cuda.synchronize()
    assert torch.equal(slot, flat)
    wm = L.new_arena(dev)
    for bad in (1.0, -0.5, 2.0):
        with pytest.raises(ValueError, match=r"\[0, 1\)"):
            K.push_encode(L, [g32], [g16], slot, step_ptr=push.step, worker=2, done_counter=push.cnt, wmom=wm, wm_beta=bad)
    with pytest.raises(ValueError, match="cyclic"):
        K.push_encode(L, [g32], [g16], slot, step_ptr=push.step, worker=2, done_counter=push.cnt, coef=[1.0], wmom=wm,
                      wm_beta=0.5)
    assert float(wm.abs().sum()) == 0


# ------------------------------------------------------------------------------------------------ engine
def _cfg(**kw):
    base = dict(network="LeNet", dataset="MNIST", batch_size=16, max_steps=12, num_workers=7, transport="nvl", lr=0.02,
                momentum=0.0, synthetic_size=512, eval_freq=10 ** 6, compress_grad="None", dtype="fp32", cuda_graphs=False,
                worker_momentum=BETA)
    base.update(kw)
    return JobConfig(**base)


def _run(cfg, steps):
    t = Trainer(cfg, rank=0, world=1, device=torch.device("cuda", 0), quiet=True)
    losses = [t.train_step()["loss"] for _ in range(steps)]
    t.synchronize()
    return t, losses


@pytest.mark.parametrize("kw", [dict(approach="baseline", mode="normal", worker_fail=0, err_mode="none"),
                                dict(approach="baseline", mode="coordinate_median", worker_fail=2, err_mode="rev_grad"),
                                dict(approach="baseline", mode="multi_krum", worker_fail=1, err_mode="constant"),
                                dict(approach="maj_vote", mode="maj_vote", group_size=3, worker_fail=1, err_mode="rev_grad"),
                                dict(approach="detox", mode="coordinate_median", num_workers=9, group_size=3, worker_fail=1,
                                     err_mode="rev_grad")])
def test_fused_matches_library_op_engine(monkeypatch, kw):
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    a, _ = _run(_cfg(**kw), 4)
    b, _ = _run(_cfg(transport="nccl", **kw), 4)
    pa, pb = a.engine.master_params(), b.engine.master_params()
    assert torch.isfinite(pa).all()
    assert torch.allclose(pa, pb, atol=2e-5), float((pa - pb).abs().max())
    for w in range(1, a.engine.P + 1):
        ma, mb = a.engine.worker_momentum[w], b.engine.worker_momentum[w]
        assert float(ma.abs().max()) > 0
        assert torch.allclose(ma, mb, atol=2e-5), (w, float((ma - mb).abs().max()))


_RESNET = dict(network="ResNet18", dataset="Cifar10", batch_size=8, num_workers=3, dtype="bf16", synthetic_size=256,
               approach="maj_vote", mode="maj_vote", group_size=3, worker_fail=1, err_mode="rev_grad", momentum=0.5)


def test_graph_replay_equals_eager_and_launches_no_extra_kernel():
    e, le = _run(_cfg(cuda_graphs=False, **_RESNET), 6)
    g, lg = _run(_cfg(cuda_graphs=True, **_RESNET), 6)
    assert g.engine.graph is not None
    assert torch.equal(e.engine.master_params(), g.engine.master_params()) and le == lg
    for w in (1, 2, 3):                                         # the state advanced exactly once per replayed step
        assert torch.equal(e.engine.worker_momentum[w], g.engine.worker_momentum[w])
    off, _ = _run(_cfg(cuda_graphs=True, **dict(_RESNET, worker_momentum=0.0)), 6)
    assert off.engine.worker_momentum == {} and off.engine.kernels_per_step == g.engine.kernels_per_step


@pytest.mark.parametrize("graphs", [False, True])
def test_worker_streams_are_bit_identical_to_serial(graphs):
    kw = dict(_RESNET, num_workers=7, worker_fail=2, cuda_graphs=graphs)
    a, la = _run(_cfg(worker_streams=1, **kw), 5)
    b, lb = _run(_cfg(worker_streams=3, **kw), 5)
    assert len(b.engine.worker_streams) == 3 and not a.engine.worker_streams
    assert torch.equal(a.engine.master_params(), b.engine.master_params()) and la == lb


def test_compressed_wire_equals_the_uncompressed_one():
    a, la = _run(_cfg(compress_grad="None", **_RESNET), 4)
    b, lb = _run(_cfg(compress_grad="compress", **_RESNET), 4)
    assert b.engine.compress
    assert torch.equal(a.engine.master_params(), b.engine.master_params()) and la == lb
    for w in (1, 2, 3):
        assert torch.equal(a.engine.worker_momentum[w], b.engine.worker_momentum[w])


@pytest.mark.parametrize("compress", ["None", "compress"])
def test_debug_checksum_passes_and_does_not_advance_the_state_twice(compress):
    kw = dict(_RESNET, compress_grad=compress)
    a, la = _run(_cfg(debug_checksum=True, **kw), 4)
    b, lb = _run(_cfg(cuda_graphs=False, **kw), 4)
    log = a.engine.checksum_log
    assert [r["step"] for r in log] == [1, 2, 3, 4] and all(r["checked"] == 3 and r["bad"] == [] for r in log)
    assert torch.equal(a.engine.master_params(), b.engine.master_params()) and la == lb
    for w in (1, 2, 3):
        assert torch.equal(a.engine.worker_momentum[w], b.engine.worker_momentum[w])


@pytest.mark.parametrize("mode", ["alie", "minmax"])
def test_ps_attacks_in_the_captured_step_equal_eager(mode):
    kw = dict(_RESNET, approach="baseline", mode="coordinate_median", num_workers=7, worker_fail=2, err_mode=mode)
    e, le = _run(_cfg(cuda_graphs=False, **kw), 5)
    g, lg = _run(_cfg(cuda_graphs=True, **kw), 5)
    assert g.engine.graph is not None and g.engine.ps.attack == A.attack_code(mode)
    assert torch.equal(e.engine.master_params(), g.engine.master_params()) and le == lg and all(np.isfinite(lg))


def test_fused_vote_stays_exact_with_worker_momentum():
    kw = dict(_RESNET, cuda_graphs=True)
    clean, l0 = _run(_cfg(**dict(kw, worker_fail=0, err_mode="none")), 6)
    dirty, l1 = _run(_cfg(**kw), 6)
    assert torch.equal(clean.engine.master_params(), dirty.engine.master_params()) and l0 == l1


def test_resume_is_bit_for_bit(tmp_path):
    d = str(tmp_path) + "/"
    kw = dict(_RESNET, cuda_graphs=True, train_dir=d, max_steps=6)
    t = Trainer(_cfg(eval_freq=3, **kw), rank=0, world=1, device=torch.device("cuda", 0), quiet=True)
    t.fit(6)
    t.synchronize()
    blob = load_checkpoint(d + "model_step_3")
    assert sorted(blob["worker_momentum"]) == [1, 2, 3]
    t2 = Trainer(_cfg(eval_freq=10 ** 6, checkpoint_step=3, **kw), rank=0, world=1, device=torch.device("cuda", 0), quiet=True)
    for _ in range(3):
        t2.train_step()
    t2.synchronize()
    assert torch.equal(t2.engine.master_params(), t.engine.master_params())
    for w in (1, 2, 3):
        assert torch.equal(t2.engine.worker_momentum[w], t.engine.worker_momentum[w])
