"""A multi-rank solver on however many GPUs are visible: W processes of `python -m kangaroo_b200.solver`, each with the
torch.distributed environment torchrun would give it.  run_ranks puts every rank on device 0 over gloo (KGX_DIST_BACKEND), so
the multi-rank paths (the gather, the sharded exchange, the herd gather and the resume scatter) run on one GPU; solver_on
keeps torchrun and NCCL where W GPUs are visible.  No rank outlives the call: on a timeout every rank is killed and waited for."""
import os
import socket
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def run_ranks(world, args, timeout=900):
    """W solver ranks on device 0 over gloo -> (exit codes, outputs) in rank order.  On a timeout every rank is killed and
    waited for, then subprocess.TimeoutExpired is raised with what each rank printed."""
    port = free_port()
    procs, logs = [], []
    try:
        for r in range(world):
            env = dict(os.environ, RANK=str(r), WORLD_SIZE=str(world), LOCAL_RANK="0", LOCAL_WORLD_SIZE=str(world),
                       MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), KGX_DIST_BACKEND="gloo")
            log = tempfile.TemporaryFile(mode="w+")                 # a file, not a pipe: a chatty rank never blocks
            logs.append(log)
            procs.append(subprocess.Popen([sys.executable, "-m", "kangaroo_b200.solver"] + list(args), stdout=log,
                                          stderr=subprocess.STDOUT, cwd=ROOT, env=env))
        deadline = time.monotonic() + timeout
        timed_out = False
        for p in procs:
            try:
                p.wait(timeout=max(0.0, deadline - time.monotonic()))
            except subprocess.TimeoutExpired:
                timed_out = True
                break
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
        for p in procs:
            p.wait()
    outs = []
    for log in logs:
        log.seek(0)
        outs.append(log.read())
        log.close()
    if timed_out:
        raise subprocess.TimeoutExpired(["kangaroo_b200.solver"] + list(args), timeout,
                                        output="".join("--- rank %d ---\n%s" % (r, o[-2000:]) for r, o in enumerate(outs)))
    return [p.returncode for p in procs], outs


def solver_on(world, args, timeout=900):
    """the solver on W ranks -> (exit code, output): torchrun and NCCL on W GPUs where that many are visible, else W ranks
    sharing device 0 over gloo (the exit code is the first non-zero one, the outputs are joined in rank order)"""
    import torch
    if torch.cuda.device_count() >= world:
        p = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nproc-per-node", str(world), "-m",
                            "kangaroo_b200.solver"] + list(args), capture_output=True, text=True, timeout=timeout, cwd=ROOT)
        return p.returncode, p.stdout + p.stderr
    rcs, outs = run_ranks(world, args, timeout)
    return next((rc for rc in rcs if rc != 0), 0), "".join(outs)
