#!/usr/bin/env python
"""Cluster manager (parity: ``/root/reference/tools/pytorch_ec2.py``).

The reference provisions EC2 spot instances with boto3 and drives them over
paramiko (``command_map`` at pytorch_ec2.py:938-951).  An H100 deployment is a
fixed set of HGX nodes, so "provisioning" becomes inventory: the same command
names operate on a host list (``--hosts a,b,c``, a hostfile, or ``SLURM_NODELIST``
expanded by the scheduler) over ssh (paramiko), or on ``localhost`` directly.

    python tools/cluster.py get_hosts --hosts n1,n2      # writes hosts / hosts_alias / hosts_address
    python tools/cluster.py list_idle_instances          # nodes whose GPUs are idle
    python tools/cluster.py run_command "nvidia-smi -L"
    python tools/cluster.py launch                       # verify nodes are reachable and have 8 GPUs
    python tools/cluster.py clean_launch_and_run         # kill stale jobs, then launch the configured command
    python tools/cluster.py kill_all_python              # stop the jobs THIS tool started (PID files)
"""
from __future__ import annotations

import argparse
import os
import shlex
import subprocess
import sys
from typing import Dict, List, Tuple


class Cfg(dict):
    """Self-interpolating config dict (pytorch_ec2.py:12-20): values may
    reference other keys with ``%(key)s``."""

    def __getitem__(self, item):
        value = dict.__getitem__(self, item)
        if isinstance(value, str):
            seen = 0
            while "%(" in value and seen < 8:
                value = value % self
                seen += 1
        return value


cfg = Cfg({
    "name": "atomo_b200",
    "ssh_user": os.environ.get("USER", "root"),
    "ssh_key": os.path.expanduser("~/.ssh/id_rsa"),
    "repo_dir": "~/atomo_b200",
    "gpus_per_node": 8,
    "master_port": 29500,
    "nfs_server": "",
    "nfs_export": "/shared",
    "nfs_mount_point": "~/shared",
    "pid_dir": "/tmp/atomo_b200_pids",
    "train_cmd": ("cd %(repo_dir)s && python -m torch.distributed.run --nnodes=%(nnodes)s --node-rank=%(node_rank)s "
                  "--nproc-per-node %(gpus_per_node)s --master-addr %(master_addr)s --master-port %(master_port)s "
                  "-m atomo_b200.distributed_nn --backend p2p --network ResNet18 --dataset Cifar10 --code svd "
                  "--svd-rank 3 --enable-gpu=1 --train-dir %(nfs_mount_point)s/models/"),
    "nnodes": 1, "node_rank": 0, "master_addr": "127.0.0.1",
})


def _hosts(args) -> List[str]:
    if args.hosts:
        return [h for h in args.hosts.split(",") if h]
    if args.hostfile and os.path.exists(args.hostfile):
        return [l.split()[0] for l in open(args.hostfile) if l.strip() and not l.startswith("#")]
    if os.environ.get("SLURM_JOB_NODELIST"):
        out = subprocess.run(["scontrol", "show", "hostnames", os.environ["SLURM_JOB_NODELIST"]],
                             capture_output=True, text=True)
        if out.returncode == 0:
            return out.stdout.split()
    return ["localhost"]


def _run(host: str, command: str, timeout: float = 120.0) -> Tuple[int, str]:
    if host in ("localhost", "127.0.0.1"):
        r = subprocess.run(command, shell=True, capture_output=True, text=True, timeout=timeout)
        return r.returncode, r.stdout + r.stderr
    try:
        import paramiko
    except Exception:
        r = subprocess.run(["ssh", "-o", "StrictHostKeyChecking=no", host, command], capture_output=True, text=True,
                           timeout=timeout)
        return r.returncode, r.stdout + r.stderr
    client = paramiko.SSHClient()
    client.set_missing_host_key_policy(paramiko.AutoAddPolicy())
    client.connect(host, username=cfg["ssh_user"], key_filename=cfg["ssh_key"], timeout=20)
    try:
        _, out, err = client.exec_command(command, timeout=timeout)
        text = out.read().decode() + err.read().decode()
        return out.channel.recv_exit_status(), text
    finally:
        client.close()


def get_hosts(args):
    """Write ``hosts`` (ip alias), ``hosts_alias`` and ``hosts_address`` (one per rank-0..N-1 node),
    the three files the reference's ``get_hosts`` produces (pytorch_ec2.py:656-819)."""
    hosts = _hosts(args)
    here = os.path.dirname(os.path.abspath(__file__))
    with open(os.path.join(here, "hosts"), "w") as f1, open(os.path.join(here, "hosts_alias"), "w") as f2, \
            open(os.path.join(here, "hosts_address"), "w") as f3:
        for i, h in enumerate(hosts):
            alias = "deeplearning-worker%d" % (i + 1)
            f1.write("%s %s\n" % (h, alias))
            f2.write(alias + "\n")
            f3.write(h + "\n")
    print("wrote hosts/hosts_alias/hosts_address for %d node(s); node 0 hosts the parameter server" % len(hosts))
    return hosts


def _gpu_state(host: str) -> Dict[str, int]:
    rc, out = _run(host, "nvidia-smi --query-gpu=utilization.gpu,memory.used --format=csv,noheader,nounits")
    if rc != 0:
        return {"gpus": 0, "busy": 0}
    rows = [l.split(",") for l in out.strip().splitlines() if "," in l]
    busy = sum(1 for u, m in rows if int(u) > 5 or int(m) > 1024)
    return {"gpus": len(rows), "busy": busy}


def list_idle_instances(args):
    for h in _hosts(args):
        s = _gpu_state(h)
        if s["gpus"] and s["busy"] == 0:
            print("%s idle (%d GPUs)" % (h, s["gpus"]))


def list_running_instances(args):
    for h in _hosts(args):
        s = _gpu_state(h)
        print("%s %s (%d/%d GPUs busy)" % (h, "running" if s["busy"] else "idle", s["busy"], s["gpus"]))


def launch(args):
    ok = True
    for h in _hosts(args):
        s = _gpu_state(h)
        good = s["gpus"] >= 1
        ok &= good
        print("%s: %s (%d GPUs)" % (h, "ready" if good else "UNREACHABLE / no GPU", s["gpus"]))
    return ok


def run_command(args):
    for h in _hosts(args):
        rc, out = _run(h, args.command)
        print("---- %s (rc=%d)\n%s" % (h, rc, out))


def _start_job(host: str, command: str):
    pid_dir = cfg["pid_dir"]
    wrapped = ("mkdir -p %s && (setsid nohup bash -lc %s > %s/job.log 2>&1 & echo $! > %s/job.pid)"
               % (pid_dir, shlex.quote(command), pid_dir, pid_dir))
    return _run(host, wrapped)


def kill_all_python(args):
    """Stop the jobs this tool started: kill the recorded process GROUP (never by name pattern)."""
    for h in _hosts(args):
        rc, out = _run(h, "test -f %s/job.pid && kill -- -$(cat %s/job.pid) ; rm -f %s/job.pid" %
                       (cfg["pid_dir"], cfg["pid_dir"], cfg["pid_dir"]))
        print("%s: stopped (rc=%d)" % (h, rc))


kill_python = kill_all_python


def shutdown(args):
    kill_all_python(args)
    print("nodes are fixed inventory: nothing to terminate (reference: EC2 terminate, pytorch_ec2.py:370-372)")


def setup_nfs(args):
    """Mount the shared checkpoint directory on every node (pytorch_ec2.py:880-900): the evaluator
    and the PS only share files through ``--train-dir``."""
    if not cfg["nfs_server"]:
        print("set cfg['nfs_server'] (or use a pre-mounted shared filesystem)")
        return
    cmd = "mkdir -p %(nfs_mount_point)s && sudo mount -t nfs %(nfs_server)s:%(nfs_export)s %(nfs_mount_point)s" % cfg
    for h in _hosts(args):
        rc, out = _run(h, cmd)
        print("%s: rc=%d %s" % (h, rc, out.strip()))


def clean_launch_and_run(args):
    kill_all_python(args)
    hosts = _hosts(args)
    cfg["nnodes"], cfg["master_addr"] = len(hosts), hosts[0]
    for i, h in enumerate(hosts):
        cfg["node_rank"] = i
        rc, out = _start_job(h, args.command or cfg["train_cmd"])
        print("%s: started node_rank %d (rc=%d)" % (h, i, rc))


command_map = {
    "launch": launch, "get_hosts": get_hosts, "shutdown": shutdown, "kill_all_python": kill_all_python,
    "kill_python": kill_python, "run_command": run_command, "setup_nfs": setup_nfs,
    "list_idle_instances": list_idle_instances, "list_running_instances": list_running_instances,
    "clean_launch_and_run": clean_launch_and_run,
}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("cmd", choices=sorted(command_map))
    ap.add_argument("command", nargs="?", default="")
    ap.add_argument("--hosts", default="")
    ap.add_argument("--hostfile", default=os.path.join(os.path.dirname(os.path.abspath(__file__)), "hosts_address"))
    args = ap.parse_args(argv)
    return command_map[args.cmd](args)


if __name__ == "__main__":
    main()
