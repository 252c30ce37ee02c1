"""End-to-end tests of the fused (nvl) engine on one GPU (all logical ranks packed on cuda:0) and, when several GPUs are
visible, across processes over peer memory."""
import json
import os
import subprocess
import sys

import pytest
import torch

from draco_b200 import JobConfig
from draco_b200.parallel.trainer import Trainer

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cfg(**kw):
    base = dict(network="LeNet", dataset="MNIST", batch_size=16, max_steps=12, num_workers=7, transport="nvl", lr=0.02,
                momentum=0.9, synthetic_size=512, eval_freq=10 ** 6, compress_grad="None", dtype="fp32", cuda_graphs=False)
    base.update(kw)
    return JobConfig(**base)


def _run(cfg, steps, device=None):
    dev = device or torch.device("cuda", 0)
    t = Trainer(cfg, rank=0, world=1, device=dev, quiet=True)
    losses = [t.train_step()["loss"] for _ in range(steps)]
    t.synchronize()
    return t, losses


def test_fused_vote_tolerates_adversaries_bitwise():
    clean, l0 = _run(_cfg(approach="maj_vote", mode="maj_vote", group_size=7, worker_fail=0, err_mode="none"), 5)
    dirty, l1 = _run(_cfg(approach="maj_vote", mode="maj_vote", group_size=7, worker_fail=3, err_mode="rev_grad"), 5)
    assert torch.equal(clean.engine.master_params(), dirty.engine.master_params())
    assert l0 == l1
    mean, _ = _run(_cfg(approach="maj_vote", mode="normal", group_size=7, worker_fail=3, err_mode="rev_grad"), 5)
    assert not torch.allclose(clean.engine.master_params(), mean.engine.master_params(), atol=1e-3)


def test_fused_matches_library_op_engine(monkeypatch):
    """Same job through the kernels and through the torch-op PS (nccl transport on one process = no collectives).  The fp32
    model runs in true fp32: TF32 convolutions would round the two runs' worker gradients differently."""
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    for kw in (dict(approach="maj_vote", mode="maj_vote", group_size=3, worker_fail=1, err_mode="rev_grad"),
               dict(approach="baseline", mode="normal", worker_fail=0, err_mode="none"),
               dict(approach="baseline", mode="krum", worker_fail=2, err_mode="constant"),
               dict(approach="cyclic", worker_fail=2, err_mode="constant"),
               dict(approach="maj_vote", mode="maj_vote", group_size=3, worker_fail=1, err_mode="rev_grad", optimizer="adam", lr=1e-3),
               dict(approach="baseline", mode="normal", worker_fail=0, err_mode="none", optimizer="adam", amsgrad=True, lr=1e-3,
                    weight_decay=1e-4)):
        a, la = _run(_cfg(**kw), 4)
        b, lb = _run(_cfg(transport="nccl", **kw), 4)
        pa, pb = a.engine.master_params(), b.engine.master_params()
        tol = 5e-4 if kw["approach"] == "cyclic" else 2e-5
        assert torch.allclose(pa, pb, atol=tol), (kw, float((pa - pb).abs().max()))


def test_fused_transport_honours_compress_grad_losslessly():
    """--compress-grad compress on the fused transport (reference default: blosc on every gradient message,
    src/compress_gradient.py:7-15): encode locally, pack on the device, push only the packed bytes, unpack at the PS.  The codec is
    lossless, so the job is bit-identical to the uncompressed one -- for the repetition code and for the complex cyclic codewords."""
    for kw in (dict(approach="maj_vote", mode="maj_vote", group_size=3, worker_fail=1, err_mode="rev_grad"),
               dict(approach="cyclic", worker_fail=2, err_mode="constant")):
        a, la = _run(_cfg(compress_grad="None", **kw), 4)
        b, lb = _run(_cfg(compress_grad="compress", **kw), 4)
        assert b.engine.compress and torch.equal(a.engine.master_params(), b.engine.master_params()) and la == lb
        sizes = b.engine.stage_bytes.tolist()
        raw = b.engine.layout.total * b.engine.esize
        assert all(0 < s <= b.engine.codec.capacity for s in sizes) and min(sizes) < raw, (sizes, raw)
    # graph capture: the packed size lives on the device, nothing in the path synchronises with the host
    g, lg = _run(_cfg(compress_grad="compress", cuda_graphs=True, approach="maj_vote", mode="maj_vote", group_size=3, worker_fail=1,
                      err_mode="rev_grad"), 6)
    e, le = _run(_cfg(compress_grad="None", cuda_graphs=False, approach="maj_vote", mode="maj_vote", group_size=3, worker_fail=1,
                      err_mode="rev_grad"), 6)
    assert g.engine.graph is not None and torch.equal(g.engine.master_params(), e.engine.master_params()) and lg == le


def test_fused_cyclic_and_geomedian_tolerate_adversaries():
    clean, _ = _run(_cfg(approach="cyclic", worker_fail=2, err_mode="none"), 4)
    dirty, _ = _run(_cfg(approach="cyclic", worker_fail=2, err_mode="rev_grad"), 4)
    a, b = clean.engine.master_params(), dirty.engine.master_params()
    assert torch.allclose(a, b, atol=5e-4), float((a - b).abs().max())
    assert dirty.engine.ps.flagged.tolist() == [2] * dirty.engine.layout.ntensors
    gm, lg = _run(_cfg(approach="baseline", mode="geometric_median", worker_fail=2, err_mode="rev_grad", lr=0.05), 10)
    assert lg[-1] < lg[0] and torch.isfinite(gm.engine.master_params()).all()


def test_cuda_graph_replay_equals_eager():
    kw = dict(approach="maj_vote", mode="maj_vote", group_size=3, worker_fail=1, err_mode="rev_grad", network="ResNet18",
              dataset="Cifar10", batch_size=8, num_workers=3, dtype="bf16", synthetic_size=256)
    e, le = _run(_cfg(cuda_graphs=False, **kw), 6)
    g, lg = _run(_cfg(cuda_graphs=True, **kw), 6)
    assert g.engine.graph is not None
    assert torch.equal(e.engine.master_params(), g.engine.master_params())
    assert le == lg
    assert g.engine.kernels_per_step >= 5


def test_replicas_are_bit_identical_resnet_bf16():
    """Determinism precondition of the majority vote: two replicas of a group produce identical flat gradients."""
    kw = dict(approach="maj_vote", mode="maj_vote", group_size=2, worker_fail=0, err_mode="none", network="ResNet18",
              dataset="Cifar10", batch_size=16, num_workers=2, dtype="bf16", synthetic_size=256)
    t, _ = _run(_cfg(**kw), 2)
    D = t.engine.layout.total
    slots = t.engine.grad_in.view(2, D)
    assert torch.equal(slots[0], slots[1]) and float(slots[0].abs().sum()) > 0
    assert t.engine.ps.winner_member.abs().sum().item() == 0


def test_omniscient_attack_and_vgg_dropout_replicas():
    om, lo = _run(_cfg(approach="maj_vote", mode="maj_vote", group_size=7, worker_fail=2, err_mode="omniscient"), 3)
    cl, lc = _run(_cfg(approach="maj_vote", mode="maj_vote", group_size=7, worker_fail=0, err_mode="none"), 3)
    assert torch.equal(om.engine.master_params(), cl.engine.master_params())
    kw = dict(approach="cyclic", worker_fail=1, err_mode="constant", network="VGG11", dataset="Cifar10", batch_size=8,
              num_workers=3, dtype="bf16", synthetic_size=128, lr=0.01)
    v, lv = _run(_cfg(**kw), 3)
    assert v.engine.ps.flagged.tolist() == [1] * v.engine.layout.ntensors      # dropout masks agreed across holders
    assert all(l == l for l in lv)
    # ... and under CUDA-graph replay (capture at step 3, replays after): the mask key reads the device step counter, so honest
    # codewords stay consistent (exactly the one liar is flagged per tensor) and the run equals the eager one bit for bit
    g, lg = _run(_cfg(cuda_graphs=True, **kw), 7)
    e, le = _run(_cfg(cuda_graphs=False, **kw), 7)
    assert g.engine.graph is not None and g.engine.ps.flagged.tolist() == [1] * g.engine.layout.ntensors
    assert torch.equal(g.engine.master_params(), e.engine.master_params()) and lg == le
    # repetition code with dropout: replicas of a group agree exactly inside the replayed graph
    kv = dict(approach="maj_vote", mode="maj_vote", group_size=3, worker_fail=1, err_mode="rev_grad", network="VGG11", dataset="Cifar10",
              batch_size=8, num_workers=3, dtype="bf16", synthetic_size=128, lr=0.01)
    a, _ = _run(_cfg(cuda_graphs=True, **kv), 6)
    b, _ = _run(_cfg(cuda_graphs=True, **dict(kv, worker_fail=0, err_mode="none")), 6)
    assert torch.equal(a.engine.master_params(), b.engine.master_params())


def test_smoke_entry():
    sys.path.insert(0, ROOT)
    import __graft_entry__ as ge
    ge.smoke()


def _torchrun(nproc, env_extra=None, port=29541, timeout=900):
    env = dict(os.environ, PYTHONPATH=ROOT, **(env_extra or {}))
    script = os.path.join(ROOT, "tests", "mp_equiv.py")
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
                          "--master-addr", "127.0.0.1", "--master-port", str(port), script], capture_output=True, text=True,
                         timeout=timeout, env=env)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    return json.loads([l for l in out.stdout.splitlines() if l.startswith("{")][-1])


@pytest.mark.timeout(900)
def test_two_processes_share_one_gpu_over_peer_memory():
    """Runs on a ONE-GPU box: PS process + worker process on the same device.  The symmetric-memory runtime (VMM allocation exported
    as a POSIX fd, SCM_RIGHTS, import + map in the peer: csrc/cuda/rt_symm.cpp), the step-stamped flags and the push / vote /
    update / broadcast kernels cross a process boundary; the parameters of both processes are bit-identical to each other and to
    the same job run in a single process."""
    rec = _torchrun(2, {"DRACO_BOOTSTRAP": "gloo", "CUDA_VISIBLE_DEVICES": os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0],
                        "MP_EQUIV_CFG": json.dumps({"multicast": "off", "cuda_graphs": False}), "MP_EQUIV_STEPS": "4"}, port=29547)
    assert rec["gpus"] == 1 and rec["world"] == 2
    assert rec["sha"][0] == rec["sha"][1]                                # PS master copy == what the worker process trained on
    single, _ = _run(_cfg(approach="maj_vote", mode="maj_vote", group_size=3, worker_fail=1, err_mode="rev_grad",
                          network="ResNet18", dataset="Cifar10", batch_size=8, dtype="bf16", synthetic_size=256), 4)
    import hashlib
    assert hashlib.sha256(single.engine.master_params().cpu().numpy().tobytes()).hexdigest() == rec["sha"][0]


def _nproc():
    return min(8, torch.cuda.device_count())


_FLAGSHIP = dict(approach="maj_vote", mode="maj_vote", group_size=3, worker_fail=1, err_mode="rev_grad", network="ResNet18",
                 dataset="Cifar10", batch_size=8, dtype="bf16", synthetic_size=256)


def _sha(t):
    import hashlib
    return hashlib.sha256(t.cpu().numpy().tobytes()).hexdigest()


@pytest.mark.multigpu
@pytest.mark.timeout(900)
def test_multi_process_peer_memory_matches_single_process():
    """N GPU processes over peer memory (+ NVLS when available): EVERY rank's full parameter arena is bit-identical to the PS's,
    and to the same job packed on one GPU (placement never changes the arithmetic)."""
    rec = _torchrun(_nproc(), port=29533)
    assert len(set(rec["sha"])) == 1, rec["sha"]
    single, _ = _run(_cfg(cuda_graphs=True, **_FLAGSHIP), 6)
    assert _sha(single.engine.master_params()) == rec["sha"][0]


@pytest.mark.multigpu
@pytest.mark.timeout(900)
def test_multigpu_nvls_multicast_equals_unicast_broadcast():
    """PS -> worker broadcast through one multimem.st stream (NVLS) and through per-destination peer stores: same bits."""
    mc = _torchrun(_nproc(), {"MP_EQUIV_CFG": json.dumps({"multicast": "auto"})}, port=29534)
    uc = _torchrun(_nproc(), {"MP_EQUIV_CFG": json.dumps({"multicast": "off"})}, port=29535)
    assert not uc["multicast"] and len(set(mc["sha"] + uc["sha"])) == 1
    if not mc["multicast"]:
        pytest.skip("NVLS multicast not available on this box: only the unicast path ran")


@pytest.mark.multigpu
@pytest.mark.timeout(1200)
def test_multigpu_fused_transport_equals_nccl_transport(tmp_path):
    """Same seeds through the fused peer-memory transport and through NCCL + library-op PS (also with Adam and with the wire
    codec on): the parameters agree to fp32 round-off."""
    for i, extra in enumerate(({}, {"optimizer": "adam", "lr": 1e-3}, {"compress_grad": "compress"})):
        outs = []
        for j, tr in enumerate(("nvl", "nccl")):
            f = str(tmp_path / f"p_{i}_{tr}.pt")
            # Adam: ONE step.  Its update is lr * m / sqrt(v) -- scale-free, so after the first step every parameter has moved by
            # exactly lr * sign(g) and the transports must agree except where an aggregate is ~0.  Later steps amplify 1-ulp
            # differences of the aggregate (sum order of the group winners) through bf16 rounding in an 18-layer network: the
            # trajectories stay close (SGD: <= 5e-5 after 4 steps) but not ulp-close under a normalising optimizer.
            steps = "1" if extra.get("optimizer") == "adam" else "4"
            _torchrun(_nproc(), {"MP_EQUIV_CFG": json.dumps(dict(extra, transport=tr, cuda_graphs=(tr == "nvl"))), "MP_EQUIV_OUT": f,
                                 "MP_EQUIV_STEPS": steps}, port=29536 + 2 * i + j)
            outs.append(torch.load(f)["params"])
        diff = (outs[0] - outs[1]).abs()
        if extra.get("optimizer") == "adam":
            assert float(diff.max()) <= 2e-3 + 1e-6 and float((diff > 1e-6).float().mean()) < 1e-3, \
                (extra, float(diff.max()), float((diff > 1e-6).float().mean()))
        else:
            assert torch.allclose(outs[0], outs[1], atol=5e-5), (extra, float(diff.max()))


@pytest.mark.multigpu
@pytest.mark.timeout(900)
def test_multigpu_vote_tolerates_s_liars_but_not_more():
    """r = 3 tolerates one liar per group: with --worker-fail 1 the job equals the adversary-free job bit for bit on N GPUs; with
    3 liars drawn over 7 workers a group gets out-voted sooner or later and the parameters leave the oracle."""
    clean = _torchrun(_nproc(), {"MP_EQUIV_CFG": json.dumps({"worker_fail": 0, "err_mode": "none"})}, port=29543)
    one = _torchrun(_nproc(), {"MP_EQUIV_CFG": json.dumps({"worker_fail": 1})}, port=29544)
    three = _torchrun(_nproc(), {"MP_EQUIV_CFG": json.dumps({"worker_fail": 3}), "MP_EQUIV_STEPS": "12"}, port=29545)
    clean12 = _torchrun(_nproc(), {"MP_EQUIV_CFG": json.dumps({"worker_fail": 0, "err_mode": "none"}), "MP_EQUIV_STEPS": "12"}, port=29546)
    assert one["sha"][0] == clean["sha"][0]
    assert three["sha"][0] != clean12["sha"][0]


@pytest.mark.multigpu
@pytest.mark.timeout(900)
def test_multigpu_job_trains_under_attack():
    """200 steps on N GPUs with one sign-flip adversary per step: the loss goes down (the 8-GPU path TRAINS, not just runs)."""
    rec = _torchrun(_nproc(), {"MP_EQUIV_CFG": json.dumps({"max_steps": 210, "lr": 0.02}), "MP_EQUIV_STEPS": "200"}, port=29548)
    first = [l[0] for l in rec["losses"] if l[0] is not None]
    last = [l[1] for l in rec["losses"] if l[1] is not None]
    assert last and sum(last) / len(last) < 0.7 * sum(first) / len(first), rec["losses"]


def test_resnet50_bottlenecks_train_on_the_fused_path():
    """ResNet-50 (ImageNet-shaped model): pointwise convs on the wgmma GEMM, fused BN, r=5 vote, graph replay."""
    from draco_b200.ops.conv import backend_counters as conv_c
    from draco_b200.ops.norm import backend_counters as bn_c
    c0, b0 = conv_c["tcgen05"], bn_c["fused"]
    kw = dict(approach="maj_vote", mode="maj_vote", group_size=5, worker_fail=2, err_mode="rev_grad", network="ResNet50",
              dataset="Cifar10", batch_size=8, num_workers=5, dtype="bf16", synthetic_size=128, cuda_graphs=True)
    t, losses = _run(_cfg(**kw), 4)
    assert conv_c["tcgen05"] > c0 and bn_c["fused"] > b0
    assert all(l == l for l in losses)
    clean, _ = _run(_cfg(**dict(kw, worker_fail=0, err_mode="none")), 4)
    assert torch.equal(t.engine.master_params(), clean.engine.master_params())      # 2 liars of 5 are out-voted, bitwise


@pytest.mark.parametrize("kw", [dict(approach="maj_vote", mode="maj_vote", group_size=3, worker_fail=2, err_mode="random"),
                                dict(approach="cyclic", worker_fail=1, err_mode="constant"),
                                dict(approach="baseline", mode="geometric_median", worker_fail=2, err_mode="rev_grad")])
def test_debug_checksum_verifies_every_pushed_gradient(kw):
    """--debug-checksum: loopback re-encode on the worker vs the words that landed in the PS slot."""
    t, losses = _run(_cfg(debug_checksum=True, **kw), 4)
    log = t.engine.checksum_log
    assert [r["step"] for r in log] == [1, 2, 3, 4]
    assert all(r["checked"] == 7 and r["bad"] == [] for r in log)
    # a word flipped in a slot after the push must be caught
    eng = t.engine
    orig = eng._verify_checksums

    def corrupt_then_verify(step):
        eng._dbg_ps_sums = eng._dbg_ps_sums.clone()
        eng._dbg_ps_sums[2] += 1
        orig(step)

    eng._verify_checksums = corrupt_then_verify
    with pytest.raises(RuntimeError, match=r"checksum mismatch for worker\(s\) \[3\]"):
        t.train_step()


def test_phase_times_are_reported_every_step_in_graph_mode():
    """The reference prints Comp / Comm / Encode / Method / Update every step (src/worker/cyclic_worker.py:154-156,
    src/master/cyclic_master.py:143).  Here they come from %globaltimer stamps inside the captured step -- no --profile-phases, no
    host synchronisation -- and ride on the pipelined metric read."""
    t, _ = _run(_cfg(approach="maj_vote", mode="maj_vote", group_size=3, worker_fail=1, err_mode="rev_grad", cuda_graphs=True), 5)
    assert t.engine.graph is not None
    m = t.train_step()
    for k in ("t_fetch", "t_comp_encode_push", "t_gather", "t_decode", "t_update"):
        assert k in m and 0 <= m[k] < 5.0, (k, m)
    assert m["t_comp_encode_push"] > 0 and m["t_update"] > 0 and "loss" in m


def test_profile_phases_on_the_fused_engine():
    t, _ = _run(_cfg(approach="maj_vote", mode="maj_vote", group_size=3, worker_fail=1, err_mode="rev_grad", profile_phases=True), 1)
    m = t.train_step()
    assert m["t_fetch"] >= 0 and m["t_comp_encode_push"] > 0 and m["t_gather_decode_update_bcast"] > 0


@pytest.mark.parametrize("graphs", [False, True])
def test_concurrent_worker_streams_are_bit_identical_to_serial(graphs):
    """--worker-streams: logical workers sharing the GPU run on concurrent streams; every worker's kernel sequence is
    unchanged, so parameters after K steps equal the serial run bit for bit (eager and under CUDA-graph replay)."""
    kw = dict(approach="maj_vote", mode="maj_vote", group_size=3, worker_fail=2, err_mode="rev_grad", network="ResNet18",
              dataset="Cifar10", batch_size=16, num_workers=7, dtype="bf16", synthetic_size=256, cuda_graphs=graphs)
    a, la = _run(_cfg(worker_streams=1, **kw), 5)
    b, lb = _run(_cfg(worker_streams=3, **kw), 5)
    assert len(b.engine.worker_streams) == 3 and not a.engine.worker_streams
    assert torch.equal(a.engine.master_params(), b.engine.master_params())
    assert la == lb
    D = b.engine.layout.total
    slots = b.engine.grad_in.view(7, D)
    groups = b.engine.groups.groups
    for grp in groups:                                   # replicas of a group still agree exactly
        honest = [w for w in grp if not b.engine.schedule.is_adversary(w, 5)]
        for w in honest[1:]:
            assert torch.equal(slots[honest[0] - 1], slots[w - 1])


@pytest.mark.parametrize("graphs", [False, True])
def test_wgrad_side_stream_is_bit_identical(graphs):
    """--wgrad-stream: weight-gradient kernels forked onto a side stream overlap the rest of the backward chain; joins happen before a
    bucket is pushed and after backward.  Same kernels per tensor => same bits, eager and under graph replay."""
    from draco_b200.ops import conv as C
    kw = dict(approach="maj_vote", mode="maj_vote", group_size=3, worker_fail=1, err_mode="rev_grad", network="ResNet18",
              dataset="Cifar10", batch_size=16, num_workers=3, dtype="bf16", synthetic_size=256, cuda_graphs=graphs, worker_streams=1)
    a, la = _run(_cfg(wgrad_stream="off", **kw), 5)
    assert not C.WGRAD_SIDE_STREAM
    b, lb = _run(_cfg(wgrad_stream="on", **kw), 5)
    assert C.WGRAD_SIDE_STREAM and C._side_streams
    C.WGRAD_SIDE_STREAM = False
    assert torch.equal(a.engine.master_params(), b.engine.master_params()) and la == lb


def test_pipelined_metric_reads_return_the_same_numbers_one_step_late():
    kw = dict(approach="maj_vote", mode="maj_vote", group_size=3, worker_fail=1, err_mode="rev_grad", cuda_graphs=True)
    _, sync_losses = _run(_cfg(**kw), 6)
    t = Trainer(_cfg(**kw), rank=0, world=1, device=torch.device("cuda", 0), quiet=True)
    got = [t.train_step_pipelined() for _ in range(6)]
    assert got[0] is None
    lag = [m["loss"] for m in got[1:]] + [t.drain()["loss"]]
    assert lag == sync_losses
    assert t.drain() is None
