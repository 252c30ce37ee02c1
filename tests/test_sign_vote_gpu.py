"""signSGD with majority vote on the GPU: the sign builds of the push kernel (csrc/cuda/push_encode.cu) bit for bit against
``oracle.sign_pack`` in both gradient modes, every attack, with worker momentum, bucketed and with non-zero padding; update-kernel
mode 6 (csrc/cuda/aggregate_update.cu) against a torch restatement for P = 1 .. 32, through the shared optimizer tail, grid and
bucket invariance and the argument checks; then whole jobs on the fused engine: against the library-op engine, graph replay,
worker streams, --debug-checksum, resume, kernels per step, and more than 16 workers."""
import ctypes as C

import numpy as np
import pytest
import torch

from draco_b200 import JobConfig
from draco_b200 import _native as N
from draco_b200.codes import oracle
from draco_b200.models import build_model
from draco_b200.parallel.arena import ArenaLayout
from draco_b200.parallel.ps import hyperparams_tensor
from draco_b200.parallel.trainer import Trainer

pytestmark = pytest.mark.gpu
BETA = 0.9


@pytest.fixture(scope="module")
def K():
    from draco_b200.ops import kernels
    return kernels


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda", 0)


@pytest.fixture(scope="module", params=["resnet18_bf16", "lenet_fp32"])
def L(request):
    # ResNet-18 in bf16: bf16 convolution / linear tensors and fp32 BatchNorm tensors; LeNet all fp32.  Every tensor is padded
    # to a tile, and most tensors end inside a word
    if request.param == "lenet_fp32":
        return ArenaLayout.from_model(build_model("LeNet"), bf16=False, channels_last=True)
    return ArenaLayout.from_model(build_model("ResNet18"), bf16=True, channels_last=True)


def _grads(L, dev, seed, pad=0.0):
    """One step's gradient: fp32 arena + bf16 arena (each tensor in its own dtype, padding ``pad``), per-tensor copies for the
    zero-copy table, and the widened fp32 flat gradient (padding 0).  A few exact zeros and negative zeros are mixed in."""
    g = torch.Generator().manual_seed(seed)
    g32 = torch.full((L.total,), pad, device=dev)
    g16 = torch.full((L.total,), pad, device=dev, dtype=torch.bfloat16)
    per = []
    for s in L.specs:
        v = torch.randn(s.numel, generator=g) * 0.1
        v[::17] = 0.0
        v[5::19] = -0.0
        v = v.to(dev)
        if s.is_bf16:
            v = v.to(torch.bfloat16)
            g16[s.offset: s.offset + s.numel] = v
        else:
            g32[s.offset: s.offset + s.numel] = v
        per.append(v.clone())
    flat = L.new_arena(dev)
    for s, v in zip(L.specs, per):
        flat[s.offset: s.offset + s.numel] = v.float()
    table = torch.tensor([[v.data_ptr() for v in per]], dtype=torch.int64, device=dev)
    return g32, g16, per, table, flat


def _pack(L, x):
    return torch.from_numpy(oracle.sign_pack(x.cpu().numpy(), L.valid_mask()).view(np.int32).copy()).to(x.device)


class _Push:
    def __init__(self, K, L, dev, attack=0):
        self.K, self.L = K, L
        self.step = torch.ones(1, dtype=torch.int64, device=dev)
        self.cnt = torch.zeros(1, dtype=torch.int32, device=dev)
        self.bitmap = torch.tensor([1 << 2], dtype=torch.int32, device=dev)      # worker slot 2 lies every step
        self.attack = attack

    def __call__(self, g32, g16, dst, table=None, wmom=None, sign=True, tile_range=None, grid=None, local_copy=None):
        self.K.push_encode(self.L, [g32], [g16], dst, step_ptr=self.step, worker=2, done_counter=self.cnt,
                           adv_bitmap=self.bitmap if self.attack else None, adv_len=1 if self.attack else 0, attack=self.attack,
                           magnitude=-100.0, seed=5, src_table=table, tile_range=tile_range, grid=grid, local_copy=local_copy,
                           wmom=wmom, wm_beta=BETA if wmom is not None else 0.0, sign=sign)


@pytest.mark.parametrize("wm", [False, True])
@pytest.mark.parametrize("zero_copy", [False, True])
@pytest.mark.parametrize("attack", [0, 1, 2, 3])
def test_sign_push_equals_the_oracle_pack_of_the_plain_push(K, L, dev, wm, zero_copy, attack):
    """The sign build stores sign_pack(what the plain build stores): the plain build is the oracle's fp32 row (worker momentum,
    the adversary hook, the random attack's generator included).  The momentum state advances the same in both builds."""
    push = _Push(K, L, dev, attack)
    wm_sign, wm_plain = (L.new_arena(dev), L.new_arena(dev)) if wm else (None, None)
    m_ref = L.new_arena(dev)
    b, c = oracle.worker_momentum_coefficients(BETA)
    words = torch.zeros(L.total // 32, dtype=torch.int32, device=dev)
    copy = torch.full((L.total // 32,), 7, dtype=torch.int32, device=dev)
    plain = L.new_arena(dev)
    for step in range(1, 4):
        push.step.fill_(step)
        g32, g16, _, table, flat = _grads(L, dev, seed=10 * step + zero_copy)
        t = table if zero_copy else None
        push(g32, g16, words, table=t, wmom=wm_sign, local_copy=copy)
        push(g32, g16, plain, table=t, wmom=wm_plain, sign=False)
        torch.cuda.synchronize()
        if wm:
            m_ref.mul_(b)
            m_ref.add_(flat * c)
            assert torch.equal(wm_sign, m_ref) and torch.equal(wm_plain, m_ref), step
        x = m_ref if wm else flat
        if attack == 0:
            assert torch.equal(plain, x)
        assert torch.equal(words, _pack(L, plain)), step
        assert torch.equal(copy, words)
        if attack == 0:
            assert torch.equal(words, _pack(L, x))
        elif attack == 1:                                      # rev_grad flips every nonzero sign
            assert torch.equal(words, _pack(L, x * -100.0))
        elif attack == 2:                                      # constant: every valid bit 1, padding 0
            assert torch.equal(words, _pack(L, torch.full_like(x, -1.0)))
    assert push.cnt.item() == 0


def test_bucketed_pushes_equal_one_whole_push_and_padding_bits_are_zero(K, L, dev):
    nt = L.ntiles
    bounds = sorted({0, nt // 7, nt // 7 + 1, nt // 2, max(nt - 3, 0), nt})
    out = []
    for how in ("whole", "buckets", "grid5"):
        push = _Push(K, L, dev, attack=1)
        wm = L.new_arena(dev)
        words = torch.zeros(L.total // 32, dtype=torch.int32, device=dev)
        for step in range(1, 4):
            push.step.fill_(step)
            g32, g16, _, _, _ = _grads(L, dev, seed=step, pad=-3.0)     # arena mode with negative padding
            if how == "buckets":
                for i in range(len(bounds) - 1):
                    push(g32, g16, words, wmom=wm, tile_range=(bounds[i], bounds[i + 1]), grid=3)
            else:
                push(g32, g16, words, wmom=wm, grid=5 if how == "grid5" else None)
        torch.cuda.synchronize()
        out.append((wm, words))
    for wm, words in out[1:]:
        assert torch.equal(wm, out[0][0]) and torch.equal(words, out[0][1])
    bits = torch.from_numpy(oracle.sign_unpack(out[0][1].cpu().numpy().view(np.uint32)))
    assert int(bits[torch.from_numpy(~L.valid_mask())].sum()) == 0
    assert int(bits.sum()) > 0


def test_push_launcher_checks_arguments(K, dev):
    L = ArenaLayout.from_model(build_model("LeNet"), bf16=False, channels_last=True)
    push = _Push(K, L, dev)
    g32, g16, _, _, _ = _grads(L, dev, seed=3)
    words = torch.zeros(L.total // 32, dtype=torch.int32, device=dev)
    with pytest.raises(ValueError, match="cyclic"):
        K.push_encode(L, [g32], [g16], words, step_ptr=push.step, worker=2, done_counter=push.cnt, coef=[1.0], sign=True)
    a = N.PushArgs()
    a.sign, a.cyclic, a.R = 1, 1, 1
    assert N.cuda().drc_push_encode(C.byref(a), 1, K._stream()) != 0
    assert int(words.abs().sum()) == 0


# ------------------------------------------------------------------------------------------------ update (mode 6)
def _restate_vote(L, words, P, dev):
    """Torch restatement of the vote: unpack the P rows of uint32 words, count the 1 bits per coordinate."""
    shifts = torch.arange(32, device=dev, dtype=torch.int64)
    bits = ((words[:P].to(torch.int64)[:, :, None] >> shifts) & 1).reshape(P, -1)
    n_neg = bits.sum(0)
    n_pos = P - n_neg
    g = torch.where(n_pos > n_neg, 1.0, torch.where(n_neg > n_pos, -1.0, 0.0)).float()
    return torch.where(torch.from_numpy(L.valid_mask()).to(dev), g, torch.zeros_like(g))


def _sign_rows(L, P, dev, seed):
    """P rows of random sign words; rows 1 and 2 repeat row 0 in a third of the words (so even P ties there), and every padding
    bit is set (the vote must ignore it)."""
    g = torch.Generator().manual_seed(seed)
    w = torch.randint(-2 ** 31, 2 ** 31 - 1, (P, L.total // 32), generator=g, dtype=torch.int64).to(torch.int32)
    if P >= 2:
        w[1, ::3] = ~w[0, ::3]
    pad = torch.from_numpy(~L.valid_mask()).reshape(-1, 32)
    padbits = (pad.to(torch.int64) << torch.arange(32)).sum(1).to(torch.int64)
    w = (w.to(torch.int64) | padbits[None]).to(torch.int64)
    w = torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)
    return w.contiguous().to(dev)


def _state(L, dev, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(L.total, generator=g) * s).to(dev) for s in (1.0, 0.1, 0.01)]


@pytest.mark.parametrize("P", list(range(1, 33)))
def test_mode6_equals_the_torch_restatement(K, dev, P):
    L = ArenaLayout.from_model(build_model("LeNet"), bf16=False, channels_last=True)
    words = _sign_rows(L, P, dev, seed=P)
    want = _restate_vote(L, words, P, dev)
    params, mom, _ = _state(L, dev, P)
    p0 = params.clone()
    step, cnt = torch.ones(1, dtype=torch.int64, device=dev), torch.zeros(4, dtype=torch.int32, device=dev)
    flags = torch.zeros(2, dtype=torch.int64, device=dev)
    gout = L.new_arena(dev)
    hp = hyperparams_tensor(JobConfig(lr=0.125, momentum=0.0), dev)
    K.sign_vote_update(L, words, L.total // 32, P=P, params=params, momentum=mom, hp=hp, step_ptr=step, done_counter=cnt[0:1],
                       grad_out=gout, flags=[flags[0:1]])
    torch.cuda.synchronize()
    assert torch.equal(gout.view(torch.int32), want.view(torch.int32))        # +0 on ties and padding, never -0
    assert torch.equal(params, p0 - 0.125 * want)                             # exact: 0.125 * (+-1 | 0)
    assert int(flags[0]) == 2 and cnt[0].item() == 0
    if P % 2 == 0:
        assert int((want[:L.total][torch.from_numpy(L.valid_mask()).to(dev)] == 0).sum()) > 0
    assert torch.equal(gout, torch.from_numpy(oracle.sign_vote(oracle.sign_unpack(words.cpu().numpy().view(np.uint32)), P,
                                                               L.valid_mask())).to(dev))


@pytest.mark.parametrize("opt", [dict(momentum=0.9, weight_decay=1e-3), dict(momentum=0.9, nesterov=True),
                                 dict(optimizer="adam"), dict(optimizer="adam", amsgrad=True)])
def test_mode6_runs_the_shared_optimizer_tail(K, dev, opt):
    """Mode 6 followed by the optimizer equals mode 0 fed the restated vote as its one row, for every optimizer: the tail is
    shared."""
    L = ArenaLayout.from_model(build_model("ResNet18"), bf16=True, channels_last=True)
    P = 15
    words = _sign_rows(L, P, dev, seed=1)
    g = _restate_vote(L, words, P, dev)
    hp = hyperparams_tensor(JobConfig(lr=0.01, **opt), dev)
    adam = opt.get("optimizer") == "adam"
    outs = []
    for sign in (True, False):
        params, mom, v = _state(L, dev, 7)
        v = v.abs()
        vmax = v.clone() * 2 if opt.get("amsgrad") else None
        step, cnt = torch.ones(1, dtype=torch.int64, device=dev), torch.zeros(4, dtype=torch.int32, device=dev)
        kw = dict(params=params, momentum=mom, hp=hp, done_counter=cnt[0:1], exp_avg_sq=v if adam else None,
                  max_exp_avg_sq=vmax)
        for s in (1, 2):                                       # the first step (momentum copy) and a later one
            step.fill_(s)
            if sign:
                K.sign_vote_update(L, words, L.total // 32, P=P, step_ptr=step, **kw)
            else:
                K.aggregate_update(L, g, L.total, K=1, scale=1.0, step_ptr=step, **kw)
        torch.cuda.synchronize()
        outs.append([params, mom] + ([v] if adam else []) + ([vmax] if vmax is not None else []))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def test_mode6_does_not_depend_on_grid_or_buckets(K, dev):
    L = ArenaLayout.from_model(build_model("ResNet18"), bf16=True, channels_last=True)
    P = 31
    words = _sign_rows(L, P, dev, seed=4)
    nt = L.ntiles
    hp = hyperparams_tensor(JobConfig(lr=0.01, momentum=0.9), dev)
    res = []
    for how in ("whole", "grid1", "grid7", "buckets"):
        params, mom, _ = _state(L, dev, 3)
        gout = L.new_arena(dev)
        step, cnt = torch.ones(1, dtype=torch.int64, device=dev), torch.zeros(4, dtype=torch.int32, device=dev)
        kw = dict(P=P, params=params, momentum=mom, hp=hp, step_ptr=step, done_counter=cnt[0:1], grad_out=gout)
        if how == "buckets":
            for t0, t1 in ((0, nt // 3), (nt // 3, nt // 3 + 1), (nt // 3 + 1, nt)):
                K.sign_vote_update(L, words, L.total // 32, tile_range=(t0, t1), grid=4, **kw)
        else:
            K.sign_vote_update(L, words, L.total // 32, grid={"whole": None, "grid1": 1, "grid7": 7}[how], **kw)
        torch.cuda.synchronize()
        res.append((params, mom, gout))
    for r in res[1:]:
        assert all(torch.equal(a, b) for a, b in zip(r, res[0]))


def test_mode6_argument_checks(K, dev):
    L = ArenaLayout.from_model(build_model("LeNet"), bf16=False, channels_last=True)
    words = torch.zeros(33, L.total // 32, dtype=torch.int32, device=dev)
    params, mom, _ = _state(L, dev, 0)
    p0 = params.clone()
    hp = hyperparams_tensor(JobConfig(), dev)
    step, cnt = torch.ones(1, dtype=torch.int64, device=dev), torch.zeros(4, dtype=torch.int32, device=dev)
    kw = dict(params=params, momentum=mom, hp=hp, step_ptr=step, done_counter=cnt[0:1])
    for P in (0, 33):
        with pytest.raises(ValueError, match="1..32 rows"):
            K.sign_vote_update(L, words, L.total // 32, P=P, **kw)
    with pytest.raises(ValueError, match="uint32 words"):
        K.sign_vote_update(L, words, L.total // 32 - 1, P=3, **kw)
    lib = N.cuda()
    sel = torch.zeros(3, L.ntensors, dtype=torch.int32, device=dev)
    for K_, select in ((0, None), (33, None), (3, sel)):
        a = N.UpdateArgs()
        a.mode, a.K, a.grad_in, a.slot_stride = 6, K_, words.data_ptr(), L.total // 32
        a.select = sel.data_ptr() if select is not None else None
        assert lib.drc_aggregate_update(C.byref(a), 1, K._stream()) != 0
    torch.cuda.synchronize()
    assert torch.equal(params, p0)


# ------------------------------------------------------------------------------------------------ engine
def _cfg(**kw):
    base = dict(network="LeNet", dataset="MNIST", batch_size=16, max_steps=12, num_workers=7, transport="nvl", lr=0.002,
                momentum=0.0, synthetic_size=512, eval_freq=10 ** 6, compress_grad="None", dtype="fp32", cuda_graphs=False,
                approach="baseline", mode="sign_vote", worker_fail=3, err_mode="rev_grad")
    base.update(kw)
    return JobConfig(**base)


def _run(cfg, steps):
    t = Trainer(cfg, rank=0, world=1, device=torch.device("cuda", 0), quiet=True)
    losses = [t.train_step()["loss"] for _ in range(steps)]
    t.synchronize()
    return t, losses


@pytest.mark.parametrize("kw", [dict(), dict(worker_momentum=0.9), dict(err_mode="constant", worker_fail=2),
                                dict(num_workers=24, worker_fail=5)])
def test_fused_matches_library_op_engine(monkeypatch, kw):
    """SGD without PS momentum moves every coordinate by exactly 0 or +-lr, so the two engines agree bit for bit as long as the
    workers' gradients have the same signs."""
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    a, la = _run(_cfg(**kw), 4)
    b, lb = _run(_cfg(transport="nccl", **kw), 4)
    assert a.engine.pipeline_ps and a.engine.ps.rule == "sign_vote"
    assert a.engine.grad_in.numel() * 4 == a.engine.P * a.engine.layout.total // 8
    pa, pb = a.engine.master_params(), b.engine.master_params()
    assert torch.isfinite(pa).all() and not torch.equal(pa, a.engine.layout.new_arena(pa.device))
    assert torch.equal(pa, pb), int((pa != pb).sum())


_RESNET = dict(network="ResNet18", dataset="Cifar10", batch_size=8, num_workers=7, dtype="bf16", synthetic_size=256,
               momentum=0.5)


@pytest.mark.parametrize("kw", [dict(), dict(worker_momentum=0.9, momentum=0.0), dict(optimizer="adam", lr=1e-4)])
def test_graph_replay_equals_eager_with_the_kernels_of_the_normal_job(kw):
    e, le = _run(_cfg(cuda_graphs=False, **dict(_RESNET, **kw)), 5)
    g, lg = _run(_cfg(cuda_graphs=True, **dict(_RESNET, **kw)), 5)
    assert g.engine.graph is not None and g.engine.pipeline_ps
    assert torch.equal(e.engine.master_params(), g.engine.master_params()) and le == lg and all(np.isfinite(lg))
    normal, _ = _run(_cfg(cuda_graphs=True, **dict(_RESNET, **dict(kw, mode="normal"))), 5)
    assert normal.engine.kernels_per_step == g.engine.kernels_per_step
    assert e.engine.kernels_per_step == normal.engine.kernels_per_step == g.engine.kernels_per_step


@pytest.mark.parametrize("graphs", [False, True])
def test_worker_streams_are_bit_identical_to_serial(graphs):
    kw = dict(_RESNET, cuda_graphs=graphs, worker_momentum=0.9)
    a, la = _run(_cfg(worker_streams=1, **kw), 4)
    b, lb = _run(_cfg(worker_streams=3, **kw), 4)
    assert len(b.engine.worker_streams) == 3 and not a.engine.worker_streams
    assert torch.equal(a.engine.master_params(), b.engine.master_params()) and la == lb


@pytest.mark.parametrize("wm", [0.0, 0.9])
def test_debug_checksum_compares_the_packed_words_and_passes(wm):
    kw = dict(_RESNET, worker_momentum=wm)
    a, la = _run(_cfg(debug_checksum=True, **kw), 3)
    b, lb = _run(_cfg(cuda_graphs=False, **kw), 3)
    assert a.engine._dbg_buf.numel() == a.engine.layout.total // 32
    log = a.engine.checksum_log
    assert [r["step"] for r in log] == [1, 2, 3] and all(r["checked"] == 7 and r["bad"] == [] for r in log)
    assert torch.equal(a.engine.master_params(), b.engine.master_params()) and la == lb


def test_resume_is_bit_for_bit(tmp_path):
    d = str(tmp_path) + "/"
    kw = dict(_RESNET, cuda_graphs=True, train_dir=d, max_steps=6, worker_momentum=0.9, momentum=0.5)
    t = Trainer(_cfg(eval_freq=3, **kw), rank=0, world=1, device=torch.device("cuda", 0), quiet=True)
    t.fit(6)
    t.synchronize()
    t2 = Trainer(_cfg(eval_freq=10 ** 6, checkpoint_step=3, **kw), rank=0, world=1, device=torch.device("cuda", 0), quiet=True)
    for _ in range(3):
        t2.train_step()
    t2.synchronize()
    assert torch.equal(t2.engine.master_params(), t.engine.master_params())
    for w in range(1, 8):
        assert torch.equal(t2.engine.worker_momentum[w], t.engine.worker_momentum[w])


@pytest.mark.parametrize("f", [3, 15])
def test_more_than_16_workers_run_on_nvl(f):
    t, losses = _run(_cfg(num_workers=32, worker_fail=f, cuda_graphs=True, lr=0.005, worker_momentum=0.9), 10)
    assert t.engine.P == 32 and t.engine.graph is not None and t.engine.pipeline_ps
    assert torch.isfinite(t.engine.master_params()).all() and all(np.isfinite(losses))
    if f == 3:
        assert min(losses[-3:]) < losses[0], losses
