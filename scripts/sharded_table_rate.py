"""--dp-table sharded against --dp-table device on the solver itself, at the default grid: per step, the time from the
collected launch to the records handed to the ingest thread (sharded: partition + count all_gather + all_to_all; device: the
DPGather to rank 0, or nothing on one GPU), the ingest threads' insert time, the step time, the default capacity (the sum of
the shards'), and the time of a mid-run save with kangaroos and of a resume from it.  The key of in80.txt is not found in
the steps run, so every run does the same work.  Prints the card name and power limit, one JSON line per table, and writes
results/sharded_table_rate_W<world>.json on rank 0.

    python scripts/sharded_table_rate.py --dp 12 --steps 200
    torchrun --nproc-per-node 8 scripts/sharded_table_rate.py --dp 14 --steps 200"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def measure(table, a, start, end, pub, tmp):
    from kangaroo_b200 import solver as S
    path = os.path.join(tmp, "%s.work" % table)
    s = S.Solver(start, end, pub, a.dp, seed=1, save_work=path, save_kangaroos=True, dp_table=table)
    handoff = []
    gather = s._gather

    def timed(n_found):
        t0 = time.perf_counter()
        gather(n_found)
        handoff.append(time.perf_counter() - t0)

    s._gather = timed
    s.run(a.steps, verbose=False)
    row = dict(table=table, world=s.world, dp=a.dp, kangaroos_per_gpu=s.eng.nbKangaroo, steps=s.steps,
               handoff_ms_median=1e3 * float(np.median(handoff[8:] or handoff)), step_ms_median=1e3 * float(np.median(s._step_times[8:])),
               ingest_ms_per_step=1e3 * s.t_ingest / max(s.steps, 1), entries=s.table_entries(),
               capacity=sum(s.shard_caps) if s.sharded else (s.dps.capacity if s.rank == 0 else None),
               save_mb=s.saves[-1][0] if s.saves else None, save_s=s.saves[-1][1] if s.saves else None)
    s.close()
    t0 = time.perf_counter()
    r = S.Solver(start, end, pub, a.dp, seed=2, resume=path, dp_table=table)
    row["resume_s"] = time.perf_counter() - t0
    r.close()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dp", type=int, default=12)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--config", default=os.path.join(ROOT, "tests", "golden", "in80.txt"))
    a = ap.parse_args()
    from kangaroo_b200 import ecmath as ec
    start, end, pubs = ec.parse_config(a.config)
    rank = int(os.environ.get("RANK", "0"))
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        if int(os.environ.get("WORLD_SIZE", "1")) > 1:
            import torch.distributed as dist
            box = [tmp]
            import torch
            torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
            dist.init_process_group("nccl", device_id=torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0"))))
            dist.broadcast_object_list(box, 0)                 # one directory for every rank's pieces
            tmp = box[0]
        for table in ("device", "sharded"):
            row = measure(table, a, start, end, pubs[0], tmp)
            if rank == 0:
                row["card"] = card()
                print(json.dumps(row), flush=True)
                rows.append(row)
    if rank == 0:
        os.makedirs(os.path.join(ROOT, "results"), exist_ok=True)
        with open(os.path.join(ROOT, "results", "sharded_table_rate_W%d.json" % rows[0]["world"]), "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
