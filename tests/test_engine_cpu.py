"""CPU runtime tests: single-process collective engine for every approach, multi-process Gloo job (LeNet/MNIST),
checkpoint / resume / evaluator, CLI flag surface."""
import argparse
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from draco_b200 import JobConfig
from draco_b200.config import add_fit_args, config_from_args
from draco_b200.data import BatchPlan, augment_cifar, load_dataset, synthetic_dataset
from draco_b200.parallel.placement import Placement
from draco_b200.parallel.trainer import Trainer


def _cfg(**kw):
    base = dict(network="LeNet", dataset="MNIST", batch_size=16, max_steps=8, num_workers=7, transport="gloo", lr=0.02,
                momentum=0.9, synthetic_size=512, eval_freq=10 ** 6, compress_grad="None")
    base.update(kw)
    return JobConfig(**base)


def _run(cfg, steps):
    t = Trainer(cfg, rank=0, world=1, device=torch.device("cpu"), quiet=True)
    losses = [t.train_step()["loss"] for _ in range(steps)]
    return t, losses


def test_reference_flag_surface():
    ap = add_fit_args(argparse.ArgumentParser())
    a = ap.parse_args([])
    # names + defaults of src/distributed_nn.py:23-77
    expected = dict(batch_size=128, test_batch_size=100, max_steps=10000, epochs=100, lr=0.01, momentum=0.5, no_cuda=False,
                    seed=1, log_interval=10, network="LeNet", mode="normal", dataset="MNIST", comm_type="Bcast",
                    err_mode="rev_grad", approach="maj_vote", num_aggregate=5, eval_freq=50, train_dir="output/models/",
                    adversarial=1, worker_fail=2, group_size=5, compress_grad="compress", checkpoint_step=0)
    for k, v in expected.items():
        assert getattr(a, k) == v, k
    cfg = config_from_args(ap.parse_args(["--approach", "cyclic", "--worker-fail", "2", "--no-cuda"])).resolve(8)
    assert cfg.num_workers == 7 and cfg.transport == "gloo" and cfg.redundancy == 5
    with pytest.raises(ValueError):
        config_from_args(ap.parse_args(["--compress-grad", "zip"])).resolve(8)
    with pytest.raises(ValueError):
        config_from_args(ap.parse_args(["--approach", "cyclic", "--worker-fail", "4"])).resolve(8)


def test_placement_packs_logical_ranks():
    assert Placement(7, 8).proc_of == {0: 0, 1: 1, 2: 2, 3: 3, 4: 4, 5: 5, 6: 6, 7: 7}
    p4 = Placement(7, 4)
    assert [len(p4.local_workers(i)) for i in range(4)] == [1, 2, 2, 2]
    p2 = Placement(7, 2)
    assert [len(p2.local_workers(i)) for i in range(2)] == [3, 4]
    assert Placement(7, 1).local_workers(0) == [1, 2, 3, 4, 5, 6, 7]


def test_batch_plans_give_identical_batches_to_holders():
    ds = synthetic_dataset("MNIST", 256)
    from draco_b200.codes.repetition import group_assign
    g = group_assign(7, 3)
    plan = BatchPlan("maj_vote", len(ds), 8, 7, g.rank_to_group, g.seeds)
    for step in (1, 2, 40):
        assert np.array_equal(plan.indices(step, 1)[0], plan.indices(step, 3)[0])
        assert not np.array_equal(plan.indices(step, 1)[0], plan.indices(step, 4)[0])
    cyc = BatchPlan("cyclic", len(ds), 8, 7, redundancy=5)
    i1, i2 = cyc.indices(3, 1), cyc.indices(3, 2)
    assert len(i1) == 5 and np.array_equal(i1[1], i2[0])         # batch 1 is worker 1's 2nd and worker 2's 1st
    assert cyc.batch_ids(3, 6) == [5, 6, 0, 1, 2]
    base = BatchPlan("baseline", len(ds), 8, 7)
    assert not np.array_equal(base.indices(1, 1)[0], base.indices(1, 2)[0])
    a = augment_cifar(torch.randint(0, 255, (4, 3, 32, 32), dtype=torch.uint8), 7)
    b = augment_cifar(torch.randint(0, 255, (4, 3, 32, 32), dtype=torch.uint8), 7)
    assert a.shape == (4, 3, 32, 32) and a.dtype == torch.uint8
    x = torch.randint(0, 255, (4, 3, 32, 32), dtype=torch.uint8)
    assert torch.equal(augment_cifar(x, 5), augment_cifar(x, 5))


def test_vote_tolerates_adversaries_bitwise():
    """Training under 1 sign-flip liar per group must equal training with none, bit for bit (repetition code)."""
    # a schedule that never exceeds the group tolerance: r = 7 (one group), s = 3
    clean, _ = _run(_cfg(approach="maj_vote", mode="maj_vote", group_size=7, worker_fail=0, err_mode="none"), 5)
    dirty, _ = _run(_cfg(approach="maj_vote", mode="maj_vote", group_size=7, worker_fail=3, err_mode="rev_grad"), 5)
    assert torch.equal(clean.engine.master_params(), dirty.engine.master_params())
    # plain averaging is destroyed by the same adversaries
    mean, _ = _run(_cfg(approach="maj_vote", mode="normal", group_size=7, worker_fail=3, err_mode="rev_grad"), 5)
    assert not torch.allclose(clean.engine.master_params(), mean.engine.master_params(), atol=1e-3)


def test_cyclic_tolerates_adversaries():
    clean, l0 = _run(_cfg(approach="cyclic", worker_fail=2, err_mode="none"), 4)
    dirty, l1 = _run(_cfg(approach="cyclic", worker_fail=2, err_mode="constant"), 4)
    a, b = clean.engine.master_params(), dirty.engine.master_params()
    assert torch.allclose(a, b, atol=2e-4), float((a - b).abs().max())
    assert all(f == 2 for f in dirty.engine.ps.last_info["flagged"])
    rnd, _ = _run(_cfg(approach="cyclic", worker_fail=2, err_mode="random"), 4)
    assert torch.allclose(a, rnd.engine.master_params(), atol=2e-3)


@pytest.mark.parametrize("mode", ["normal", "krum", "geometric_median"])
def test_baseline_modes_train(mode):
    t, losses = _run(_cfg(approach="baseline", mode=mode, worker_fail=2 if mode != "normal" else 0,
                          err_mode="rev_grad" if mode != "normal" else "none", lr=0.05), 12)
    assert losses[-1] < losses[0], losses
    assert torch.isfinite(t.engine.master_params()).all()


def test_checkpoint_resume_and_evaluator(tmp_path):
    d = str(tmp_path) + "/"
    cfg = _cfg(approach="maj_vote", mode="maj_vote", group_size=7, worker_fail=0, err_mode="none", train_dir=d, eval_freq=3,
               max_steps=6)
    t = Trainer(cfg, rank=0, world=1, device=torch.device("cpu"), quiet=True)
    t.fit(6)
    assert os.path.isfile(d + "model_step_3") and os.path.isfile(d + "model_step_6")
    final = t.engine.master_params().clone()
    # resume from step 3 and replay 3 more steps -> same parameters (momentum restored, same batches)
    cfg2 = _cfg(approach="maj_vote", mode="maj_vote", group_size=7, worker_fail=0, err_mode="none", train_dir=d,
                eval_freq=10 ** 6, max_steps=6, checkpoint_step=3)
    t2 = Trainer(cfg2, rank=0, world=1, device=torch.device("cpu"), quiet=True)
    assert t2.step == 4
    from draco_b200.utils.checkpoint import load_checkpoint
    blob = load_checkpoint(d + "model_step_3")
    assert blob["step"] == 3 and len(blob["state_dict"]) == 8 and blob["config"]["network"] == "LeNet"
    assert blob["momentum"] is not None and set(blob["momentum"]) == set(blob["state_dict"])      # optimizer state is saved
    for _ in range(3):
        t2.train_step()
    assert torch.equal(t2.engine.master_params(), final)       # steps 4-6 replayed bit for bit: parameters AND momentum restored
    from draco_b200.cli.distributed_evaluator import DistributedEvaluator
    ev = DistributedEvaluator("LeNet", "MNIST", d, eval_freq=3, eval_batch_size=128, device="cpu", poll_s=0.01)
    assert ev.evaluate(max_evals=2, timeout_s=1.0) == 2


def test_adam_state_is_checkpointed_and_resumed_bit_for_bit(tmp_path):
    """--optimizer adam (reference: src/optim/adam_modified.py): first / second moment and the step count survive a
    checkpoint -- the reference saves no optimizer state at all (baseline_master.py:237-243)."""
    d = str(tmp_path) + "/"
    kw = dict(approach="baseline", mode="normal", worker_fail=0, err_mode="none", train_dir=d, optimizer="adam", amsgrad=True,
              lr=1e-3, max_steps=6)
    t = Trainer(_cfg(eval_freq=3, **kw), rank=0, world=1, device=torch.device("cpu"), quiet=True)
    t.fit(6)
    final = t.engine.master_params().clone()
    from draco_b200.utils.checkpoint import load_checkpoint
    blob = load_checkpoint(d + "model_step_3")
    assert set(blob["opt_state"]) == {"exp_avg_sq", "max_exp_avg_sq"} and blob["momentum"] is not None
    t2 = Trainer(_cfg(eval_freq=10 ** 6, checkpoint_step=3, **kw), rank=0, world=1, device=torch.device("cpu"), quiet=True)
    for _ in range(3):
        t2.train_step()
    assert torch.equal(t2.engine.master_params(), final)


def test_config_rejects_oversized_vote_groups():
    with pytest.raises(ValueError, match="members"):
        _cfg(approach="maj_vote", mode="maj_vote", group_size=5, num_workers=9, worker_fail=0, err_mode="none").resolve(1)
    _cfg(approach="maj_vote", mode="maj_vote", group_size=3, num_workers=7, worker_fail=0, err_mode="none").resolve(1)


def test_compressed_wire_roundtrip_single_proc():
    t, losses = _run(_cfg(approach="baseline", mode="normal", worker_fail=0, err_mode="none", compress_grad="compress"), 3)
    assert np.isfinite(losses).all()


# ---------------------------------------------------------------------------------------------------------------
# multi-process Gloo: LeNet/MNIST, repetition r=1, 1 PS + 2 workers, no adversary
# ---------------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _gloo_worker(rank, world, port, compress, q, comm_type="Bcast"):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    cfg = JobConfig(network="LeNet", dataset="MNIST", approach="maj_vote", mode="maj_vote", group_size=1, worker_fail=0,
                    err_mode="none", batch_size=32, max_steps=12, transport="gloo", lr=0.05, momentum=0.9, synthetic_size=512,
                    eval_freq=10 ** 6, compress_grad="compress" if compress else "None", comm_type=comm_type)
    t = Trainer(cfg, rank=rank, world=world, device=torch.device("cpu"), quiet=True)
    losses, sums = [], []
    for _ in range(12):
        m = t.train_step()
        losses.append(m.get("loss"))
        # parameters every process trained on this step (after the broadcast at the top of the step)
    t.engine._broadcast_params()
    sums.append(t.engine.master_params().double().sum().item())
    q.put((rank, losses, sums, t.engine.bytes_up, t.engine.bytes_up_raw))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("compress,comm_type", [(False, "Bcast"), (True, "Bcast"), (False, "Async")])
def test_gloo_ps_plus_two_workers(compress, comm_type):
    world, port = 3, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_worker, args=(r, world, port, compress, q, comm_type)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=240) for _ in range(world))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    (_, l0, s0, _, _), (_, l1, s1, up1, raw1), (_, l2, s2, _, _) = res
    assert l0[0] is None                                  # the PS process hosts no worker
    assert l1[-1] < l1[0] and l2[-1] < l2[0], (l1, l2)     # loss decreases on both workers
    assert s0 == s1 == s2                                 # PS / worker parameters bit-identical after the broadcast
    if compress:
        assert 0 < up1 < raw1                             # the codec actually shrank the wire volume
