"""Cluster manager -- the role of the reference's ``tools/pytorch_ec2.py`` + shell glue (tools/local_script.sh,
remote_script.sh, update_git_dir.sh, hosts*), re-thought for GPU nodes.

The reference tool rents EC2 CPU spot instances with boto3, mounts EFS, writes ``hosts`` / ``hosts_alias`` /
``hosts_address`` and fans commands out with paramiko (tools/pytorch_ec2.py:93-971; its ``Cfg`` is a dict whose string
values are interpolated against the dict itself, :12-20).  What survives here:

  * ``Cfg``                 -- the same self-interpolating config dict
  * ``get_hosts``           -- write hosts / hosts_alias / hosts_address from the configured node list, or (``--from-ec2``) from
                               the job's live instances (private address, PS first; reference :656-819)
  * ``check``               -- reachability + ``nvidia-smi`` inventory of every node (parallel fan-out)
  * ``sync``                -- push the repo to every node (rsync over ssh; replaces remote_script.sh / update_git_dir.sh)
  * ``run``                 -- start one torchrun agent per node for a draco_b200 job (replaces mpirun --hostfile)
  * ``run_command``         -- run a shell command on every node in parallel (reference :297-303, :854-878)
  * ``idle`` / ``kill``     -- find / stop running jobs (exact PIDs recorded at launch; never by pattern)
  * ``setup_nfs``           -- shared train_dir: the first node exports it over NFS (or an EFS id is mounted) on all nodes (:880-900)
  * ``launch`` / ``status`` / ``shutdown`` / ``clean_launch_and_run`` -- EC2 lifecycle through ``Ec2Fleet``: on-demand or SPOT
                               requests, wait-until-fulfilled, wait-until-running (+ status checks), summaries by state, cancel
                               requests + terminate (reference :128-257, :370-372, :905-926).  Needs boto3 (not in this image; the
                               logic is exercised in tests/test_misc_cpu.py against a stub client).

One 8-GPU H100 node hosts the whole 1 PS + 7 workers job.  ``run`` starts ONE job: on the first node, or -- with ``--nnodes`` > 1 --
spanning that many nodes through torchrun's rendezvous (the *collective* transports are used across nodes, peer memory is
intra-node).  ``run --all-nodes`` starts an independent copy on every node (sweeps), each with its own log / train_dir suffix.
"""
from __future__ import annotations

import argparse
import concurrent.futures as cf
import json
import os
import shlex
import subprocess
import sys
import time
from typing import Dict, List, Optional


class Cfg(dict):
    """dict whose string values may reference other keys as ``%(key)s`` (reference: tools/pytorch_ec2.py:12-20)."""

    def __getitem__(self, key):
        item = dict.__getitem__(self, key)
        if isinstance(item, str):
            for _ in range(8):
                new = item % self if "%(" in item else item
                if new == item:
                    break
                item = new
        return item


DEFAULT_CFG = Cfg({
    "name": "draco_b200",
    "nodes": ["127.0.0.1"],                 # hostnames / addresses of the GPU nodes
    "ssh_user": os.environ.get("USER", "root"),
    "ssh_key": "~/.ssh/id_rsa",
    "ssh_port": 22,
    "gpus_per_node": 8,
    "remote_dir": "/root/%(name)s",
    "python": sys.executable,
    "train_dir": "%(remote_dir)s/output/models/",
    "master_port": 29500,
    "state_file": ".cluster_state.json",
    # EC2 fields (Ec2Fleet)
    "region": "us-west-2", "availability_zone": "us-west-2b", "instance_type": "p5.48xlarge", "image_id": "", "key_name": "",
    "n_instances": 1, "spot_price": "", "security_group": [], "subnet_id": "", "efs_id": "", "nfs_dir": "%(remote_dir)s/output",
    "launch_timeout_s": 900, "poll_s": 5,
})


def load_cfg(path: Optional[str]) -> Cfg:
    cfg = Cfg(DEFAULT_CFG)
    if path:
        with open(path) as fh:
            cfg.update(json.load(fh))
    return cfg


def _is_local(host: str) -> bool:
    return host in ("127.0.0.1", "localhost")


def ssh_cmd(cfg: Cfg, host: str, command: str) -> List[str]:
    if _is_local(host):
        return ["bash", "-lc", command]
    return ["ssh", "-o", "StrictHostKeyChecking=no", "-o", "BatchMode=yes", "-p", str(cfg["ssh_port"]), "-i",
            os.path.expanduser(cfg["ssh_key"]), f"{cfg['ssh_user']}@{host}", command]


def run_on(cfg: Cfg, host: str, command: str, timeout: float = 60.0) -> subprocess.CompletedProcess:
    return subprocess.run(ssh_cmd(cfg, host, command), capture_output=True, text=True, timeout=timeout)


def run_parallel(cfg: Cfg, command: str, nodes: Optional[List[str]] = None, timeout: float = 60.0) -> Dict[str, dict]:
    """Run ``command`` on every node concurrently (reference: one thread per instance, run_ssh_commands_parallel :297-303)."""
    nodes = list(nodes if nodes is not None else cfg["nodes"])

    def one(n):
        try:
            r = run_on(cfg, n, command, timeout)
            return n, {"rc": r.returncode, "stdout": r.stdout, "stderr": r.stderr}
        except (subprocess.TimeoutExpired, OSError) as e:
            return n, {"rc": -1, "stdout": "", "stderr": str(e)}

    if not nodes:
        return {}
    with cf.ThreadPoolExecutor(max_workers=min(32, len(nodes))) as ex:
        return dict(ex.map(one, nodes))


def get_hosts(cfg: Cfg, out_dir: str = ".", fleet: "Optional[Ec2Fleet]" = None) -> Dict[str, str]:
    """Write ``hosts`` (addr alias), ``hosts_alias`` and ``hosts_address`` like the reference's ``get_hosts``.  With ``fleet`` the
    node list is the job's RUNNING instances (private addresses, launch order: the first one is the PS node) and is stored
    back into ``cfg["nodes"]``."""
    if fleet is not None:
        cfg["nodes"] = fleet.addresses()
    nodes = list(cfg["nodes"])
    files = {
        "hosts": "".join(f"{n}\tnode{i}\n" for i, n in enumerate(nodes)),
        "hosts_alias": "".join(f"node{i}\n" for i in range(len(nodes))),
        "hosts_address": "".join(f"{n}\n" for n in nodes),
    }
    for name, text in files.items():
        with open(os.path.join(out_dir, name), "w") as fh:
            fh.write(text)
    return files


def check(cfg: Cfg) -> Dict[str, dict]:
    out = {}
    res = run_parallel(cfg, "nvidia-smi --query-gpu=name,memory.total --format=csv,noheader || echo NO_GPU", timeout=30)
    for n, r in res.items():
        gpus = [l for l in r["stdout"].strip().splitlines() if l and "NO_GPU" not in l]
        out[n] = {"reachable": r["rc"] == 0, "gpus": gpus}
        if r["rc"] == -1:
            out[n]["error"] = r["stderr"]
    return out


def setup_nfs(cfg: Cfg) -> Dict[str, dict]:
    """Shared model / checkpoint directory (reference: setup_nfs, tools/pytorch_ec2.py:880-900 -- the PS saves checkpoints, the
    evaluator polls them from another node).  With ``efs_id`` every node mounts the EFS file system; otherwise the first node
    exports ``nfs_dir`` and the others mount it.  Idempotent (mountpoint -q)."""
    d = cfg["nfs_dir"]
    nodes = list(cfg["nodes"])
    if cfg.get("efs_id"):
        src = f"{cfg['efs_id']}.efs.{cfg['region']}.amazonaws.com:/"
        cmd = (f"mkdir -p {d} && (mountpoint -q {d} || sudo mount -t nfs4 -o nfsvers=4.1,rsize=1048576,wsize=1048576,hard,timeo=600,"
               f"retrans=2 {src} {d})")
        return run_parallel(cfg, cmd, nodes, timeout=120)
    head, rest = nodes[0], nodes[1:]
    out = {head: run_parallel(cfg, f"mkdir -p {d} && (grep -qs '^{d} ' /etc/exports || echo '{d} *(rw,sync,no_subtree_check,"
                                   f"no_root_squash)' | sudo tee -a /etc/exports) && sudo exportfs -ra", [head], timeout=120)[head]}
    out.update(run_parallel(cfg, f"mkdir -p {d} && (mountpoint -q {d} || sudo mount -t nfs {head}:{d} {d})", rest, timeout=120))
    return out


def sync(cfg: Cfg, src: str = ".") -> None:
    for n in cfg["nodes"]:
        if _is_local(n) and os.path.abspath(src) == os.path.abspath(os.path.expanduser(cfg["remote_dir"])):
            continue
        dst = cfg["remote_dir"] if _is_local(n) else f"{cfg['ssh_user']}@{n}:{cfg['remote_dir']}"
        ssh = f"ssh -p {cfg['ssh_port']} -i {os.path.expanduser(cfg['ssh_key'])} -o StrictHostKeyChecking=no"
        cmd = ["rsync", "-az", "--delete", "--exclude", ".git", "--exclude", "gpurun_out", "--exclude", "build", "-e", ssh,
               src.rstrip("/") + "/", dst]
        if _is_local(n):
            cmd = ["rsync", "-a", "--exclude", ".git", src.rstrip("/") + "/", dst]
        subprocess.run(cmd, check=True)


def job_command(cfg: Cfg, job_args: List[str], node_rank: int, nnodes: int, nproc: int) -> str:
    master = cfg["nodes"][0]
    tr = (f"{cfg['python']} -m torch.distributed.run --nnodes={nnodes} --node-rank={node_rank} --nproc-per-node={nproc} "
          f"--master-addr {master if nnodes > 1 else '127.0.0.1'} --master-port {cfg['master_port']} "
          f"-m draco_b200.cli.distributed_nn {' '.join(shlex.quote(a) for a in job_args)}")
    log = f"{cfg['remote_dir']}/job_node{node_rank}.log"
    # setsid: the agent leads its own session / process group, so ``kill`` can address exactly that group by the recorded PID
    # (the braces matter: only the agent is backgrounded, with all three standard streams redirected, so the launching shell --
    # and the ssh / subprocess pipe behind it -- returns immediately with the PID instead of waiting for the job)
    return f"cd {cfg['remote_dir']} && {{ setsid nohup {tr} > {log} 2>&1 < /dev/null & echo $!; }}"


def run(cfg: Cfg, job_args: List[str], nnodes: int = 1, nproc: Optional[int] = None, all_nodes: bool = False) -> Dict[str, int]:
    """Start ONE job on the first ``nnodes`` nodes (default: the first node); ``all_nodes`` starts an independent single-node
    copy on every node instead (sweeps; each copy logs to job_node<i>.log).  Returns {node: pid of the launched agent} and
    records it for ``idle`` / ``kill``."""
    nproc = nproc or int(cfg["gpus_per_node"])
    pids = {}
    nodes = list(cfg["nodes"]) if all_nodes else list(cfg["nodes"])[:max(nnodes, 1)]
    span = 1 if all_nodes else max(nnodes, 1)
    for i, n in enumerate(nodes):
        cmd = job_command(cfg, job_args, i if span > 1 else 0, span, nproc)
        if all_nodes:
            cmd = cmd.replace("job_node0.log", f"job_node{i}.log")
        r = run_on(cfg, n, cmd, 60)
        pids[n] = int(r.stdout.strip().splitlines()[-1]) if r.stdout.strip() else -1
    with open(cfg["state_file"], "w") as fh:
        json.dump({"pids": pids, "started": time.time(), "args": job_args}, fh)
    return pids


def idle(cfg: Cfg) -> Dict[str, bool]:
    """A node is idle when none of the recorded agent PIDs is alive (reference: idle detection via ``ps aux``)."""
    state = _state(cfg)
    res = {}
    for n in cfg["nodes"]:
        pid = state.get("pids", {}).get(n, -1)
        if pid <= 0:
            res[n] = True
            continue
        r = run_on(cfg, n, f"kill -0 {pid} 2>/dev/null && echo BUSY || echo IDLE", 30)
        res[n] = "IDLE" in r.stdout
    return res


def kill(cfg: Cfg) -> None:
    """Stop the recorded agents by exact PID / process group -- never by name pattern."""
    state = _state(cfg)
    for n, pid in state.get("pids", {}).items():
        if pid > 0:
            # the recorded PID is a process-group leader (launched under setsid): signal that group, and only that group
            run_on(cfg, n, f"kill -TERM -- -{pid} 2>/dev/null || kill -TERM {pid} 2>/dev/null; true", 30)


def _state(cfg: Cfg) -> dict:
    try:
        with open(cfg["state_file"]) as fh:
            return json.load(fh)
    except (OSError, ValueError):
        return {}


class Ec2Fleet:
    """EC2 lifecycle of a job's nodes (reference: tools/pytorch_ec2.py:128-257, 311-372).  ``client`` is a boto3 EC2 client (or
    any object with the same five methods -- the tests inject a stub; boto3 is not in this image).  Instances are found by
    their ``Name`` tag = cfg["name"]."""

    ACTIVE = ("pending", "running")

    def __init__(self, cfg: Cfg, client=None):
        self.cfg = cfg
        if client is None:
            try:
                import boto3
            except ImportError:
                raise SystemExit("boto3 is not installed in this image: EC2 launch / status / shutdown are unavailable; "
                                 "list the nodes in the config instead (\"nodes\": [...])")
            client = boto3.client("ec2", region_name=cfg["region"])
        self.ec2 = client

    # -- queries ------------------------------------------------------------------------------------------------------
    def instances(self, states=None) -> List[dict]:
        r = self.ec2.describe_instances(Filters=[{"Name": "tag:Name", "Values": [self.cfg["name"]]}])
        out = [i for res in r.get("Reservations", []) for i in res.get("Instances", [])]
        if states is not None:
            out = [i for i in out if i.get("State", {}).get("Name") in states]
        return sorted(out, key=lambda i: (str(i.get("LaunchTime", "")), i.get("InstanceId", "")))

    def summarize(self) -> Dict[str, List[str]]:
        """{state: [instance ids]} (reference: summarize_instances :100-117)."""
        out: Dict[str, List[str]] = {}
        for i in self.instances():
            out.setdefault(i.get("State", {}).get("Name", "?"), []).append(i["InstanceId"])
        return out

    def addresses(self) -> List[str]:
        return [i.get("PrivateIpAddress") or i.get("PublicIpAddress") for i in self.instances(("running",))]

    # -- lifecycle ----------------------------------------------------------------------------------------------------
    def _spec(self) -> dict:
        c = self.cfg
        spec = {"ImageId": c["image_id"], "InstanceType": c["instance_type"], "KeyName": c["key_name"]}
        if c.get("security_group"):
            spec["SecurityGroupIds"] = list(c["security_group"])
        if c.get("subnet_id"):
            spec["SubnetId"] = c["subnet_id"]
        if c.get("availability_zone"):
            spec["Placement"] = {"AvailabilityZone": c["availability_zone"]}
        return spec

    def launch(self) -> List[str]:
        """On-demand instances, or spot requests when ``spot_price`` is set (reference: launch_instances :176-207).  Returns the
        instance ids once every request is fulfilled and every instance is running with passing status checks."""
        c, n = self.cfg, int(self.cfg["n_instances"])
        have = self.instances(self.ACTIVE)
        if len(have) >= n:                                        # idempotent: a fleet of the right size already exists
            return self.wait_running([i["InstanceId"] for i in have[:n]])
        n -= len(have)
        if c.get("spot_price"):
            r = self.ec2.request_spot_instances(SpotPrice=str(c["spot_price"]), InstanceCount=n, Type="one-time",
                                                LaunchSpecification=self._spec())
            ids = self.wait_fulfilled([q["SpotInstanceRequestId"] for q in r["SpotInstanceRequests"]])
            self.ec2.create_tags(Resources=ids, Tags=[{"Key": "Name", "Value": c["name"]}])
        else:
            r = self.ec2.run_instances(MinCount=n, MaxCount=n, **self._spec(),
                                       TagSpecifications=[{"ResourceType": "instance", "Tags": [{"Key": "Name", "Value": c["name"]}]}])
            ids = [i["InstanceId"] for i in r["Instances"]]
        return self.wait_running([i["InstanceId"] for i in have] + ids)

    def _poll(self, what: str, fn):
        deadline = time.time() + float(self.cfg["launch_timeout_s"])
        while True:
            done, val = fn()
            if done:
                return val
            if time.time() > deadline:
                raise TimeoutError(f"timed out waiting for {what}: {val}")
            time.sleep(float(self.cfg["poll_s"]))

    def wait_fulfilled(self, request_ids: List[str]) -> List[str]:
        """Spot requests -> instance ids (reference: wait_until_instance_request_status_fulfilled :233-257); a request that ends
        in a terminal failed state raises instead of waiting forever."""
        def step():
            r = self.ec2.describe_spot_instance_requests(SpotInstanceRequestIds=request_ids)["SpotInstanceRequests"]
            bad = [q for q in r if q.get("State") in ("cancelled", "failed", "closed") and not q.get("InstanceId")]
            if bad:
                raise RuntimeError(f"spot request(s) not fulfilled: {[(q['SpotInstanceRequestId'], q.get('Status', {}).get('Code')) for q in bad]}")
            ids = [q.get("InstanceId") for q in r]
            return all(ids), ids
        return self._poll("spot fulfilment", step)

    def wait_running(self, instance_ids: List[str]) -> List[str]:
        """All instances 'running' with instance / system status checks 'ok' (reference: wait_until_running_instances_initialized
        :209-231)."""
        def step():
            st = self.ec2.describe_instance_status(InstanceIds=instance_ids, IncludeAllInstances=True)["InstanceStatuses"]
            ok = [s["InstanceId"] for s in st if s.get("InstanceState", {}).get("Name") == "running"
                  and s.get("InstanceStatus", {}).get("Status", "ok") in ("ok", "not-applicable")
                  and s.get("SystemStatus", {}).get("Status", "ok") in ("ok", "not-applicable")]
            return len(ok) == len(instance_ids), ok
        self._poll("instances running", step)
        return instance_ids

    def shutdown(self) -> Dict[str, List[str]]:
        """Cancel open spot requests, then terminate the job's instances (reference: terminate_all_requests / terminate_all_instances
        :128-174, shut_everything_down :370-372)."""
        reqs = []
        try:
            r = self.ec2.describe_spot_instance_requests(Filters=[{"Name": "state", "Values": ["open", "active"]}])
            mine = {i["InstanceId"] for i in self.instances()}
            reqs = [q["SpotInstanceRequestId"] for q in r.get("SpotInstanceRequests", [])
                    if q.get("InstanceId") in mine or q.get("State") == "open"]
            if reqs:
                self.ec2.cancel_spot_instance_requests(SpotInstanceRequestIds=reqs)
        except AttributeError:
            pass
        ids = [i["InstanceId"] for i in self.instances(self.ACTIVE + ("stopping", "stopped"))]
        if ids:
            self.ec2.terminate_instances(InstanceIds=ids)
        return {"cancelled_requests": reqs, "terminated": ids}


def clean_launch_and_run(cfg: Cfg, job_args: List[str], fleet: Ec2Fleet, nnodes: int = 1, out_dir: str = ".") -> Dict[str, int]:
    """shutdown -> launch -> hosts files -> sync -> shared directory -> run (reference: clean_launch_and_run :916-926)."""
    fleet.shutdown()
    fleet.launch()
    get_hosts(cfg, out_dir, fleet)
    sync(cfg)
    if len(cfg["nodes"]) > 1:
        setup_nfs(cfg)
    return run(cfg, job_args, nnodes)


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description="draco_b200 cluster manager")
    ap.add_argument("command", choices=["get_hosts", "check", "sync", "run", "run_command", "idle", "kill", "setup_nfs", "launch",
                                        "status", "shutdown", "clean_launch_and_run", "show_cfg"])
    ap.add_argument("--from-ec2", action="store_true", help="get_hosts: take the node list from the job's running EC2 instances")
    ap.add_argument("--all-nodes", action="store_true", help="run: an independent single-node copy of the job on every node")
    ap.add_argument("--config", default=None, help="JSON file overriding the default Cfg")
    ap.add_argument("--nnodes", type=int, default=1)
    ap.add_argument("--nproc-per-node", type=int, default=None)
    ap.add_argument("job_args", nargs=argparse.REMAINDER, help="flags forwarded to draco_b200.cli.distributed_nn (after --)")
    a = ap.parse_args(argv)
    cfg = load_cfg(a.config)
    job_args = [x for x in a.job_args if x != "--"]
    if a.command == "show_cfg":
        print(json.dumps({k: cfg[k] for k in cfg}, indent=1))
    elif a.command == "get_hosts":
        print(json.dumps(get_hosts(cfg, ".", Ec2Fleet(cfg) if a.from_ec2 else None)))
    elif a.command == "check":
        print(json.dumps(check(cfg), indent=1))
    elif a.command == "sync":
        sync(cfg)
    elif a.command == "run":
        print(json.dumps(run(cfg, job_args, a.nnodes, a.nproc_per_node, a.all_nodes)))
    elif a.command == "run_command":
        print(json.dumps(run_parallel(cfg, " ".join(job_args)), indent=1))
    elif a.command == "setup_nfs":
        print(json.dumps(setup_nfs(cfg), indent=1))
    elif a.command == "idle":
        print(json.dumps(idle(cfg)))
    elif a.command == "kill":
        kill(cfg)
    elif a.command == "launch":
        print(json.dumps(Ec2Fleet(cfg).launch()))
    elif a.command == "status":
        print(json.dumps(Ec2Fleet(cfg).summarize()))
    elif a.command == "shutdown":
        print(json.dumps(Ec2Fleet(cfg).shutdown()))
    else:
        print(json.dumps(clean_launch_and_run(cfg, job_args, Ec2Fleet(cfg), a.nnodes)))
    return 0


if __name__ == "__main__":
    sys.exit(main())
