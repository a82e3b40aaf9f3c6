"""End-to-end rate of the DP server with its table in shards (--devices), the counterpart of scripts/server_rate.py, whose
records, senders and clock it uses: 2^23 engine-made records (dp 8, 2^100 range), 5 % of them wrong, sent over 127.0.0.1 by 1,
4 and 8 sender processes in SENDDP messages of 2^14 records, to a server in this process (Server + GpuSink, the code
`python -m kangaroo_b200.server` runs).

Layouts: W = 1 (the one-GPU server) and W = 2, 4 and 8 GPUs, each where that many are visible (--devices 0,1,...), then W
shards on GPU 0 alone (--devices 0,0,...; --one-gpu, default 2 and 4), which measures the sharded path's own cost where
one GPU is all there is.  Per layout and sender count it prints records/s (from the first message read to the last record
inserted), the ingest thread's time per batch: host-to-device copy and verify (kgx_resolver_verify_partition) from CUDA
events, the adds from the host clock, and inside them the copies of groups to other GPUs; and the default total capacity the layout would take (each GPU's free memory at start-up split among
its shards).  Writes results/server_shards_rate.json.

    python scripts/server_shards_rate.py [--records 8388608] [--msg 16384] [--senders 1,4,8] [--one-gpu 2,4]"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import server_rate as sr                                                  # noqa: E402


def default_capacity(devices):
    """the total capacity --devices would take by default, from each GPU's free memory now"""
    import torch
    from kangaroo_b200.server import CHUNK_RECORDS, DP40, EVENT_BYTES
    from kangaroo_b200.solver import DP_TABLE_MARGIN, default_table_capacity, scratch_bytes
    per_shard = scratch_bytes(CHUNK_RECORDS) + EVENT_BYTES * CHUNK_RECORDS + (CHUNK_RECORDS * DP40 if len(set(devices)) > 1 else 0)
    total = 0
    for d in set(devices):
        k = devices.count(d)
        free = torch.cuda.mem_get_info(d)[0]
        total += k * default_table_capacity((free - DP_TABLE_MARGIN) // k - per_shard, margin=0)
    return total


def run(devices, n_send, path, total, n_wrong, msg):
    from kangaroo_b200.server import GpuSink, Server
    sink = GpuSink(sr.START, sr.END, sr.KEY, sr.DP, devices, capacity=total + (1 << 20), out=lambda s: None)
    srv = Server(sr.START, sr.END, sr.KEY, sr.DP, sink, bind="127.0.0.1", port=0, out=lambda s: None)
    srv.listen()
    first, put = [], sink.put

    def timed_put(m, chunks):                                  # the clock starts at the first message the server has read
        if not first:
            first.append(time.perf_counter())
        put(m, chunks)

    sink.put = timed_put
    try:
        procs = sr.start_senders(n_send, srv.port, path, total, msg)
        while sink.received < total and all(p.poll() in (None, 0) for p in procs) and sink.failed is None:
            time.sleep(0.001)
        t1 = time.perf_counter()
        rcs = sr.finish(procs)
    finally:
        srv.close()
        sink.finish()
    assert rcs == [0] * n_send and sink.failed is None and sink.full is None, (rcs, sink.failed, sink.full)
    assert sink.received == total and sink.wrong == n_wrong, (sink.received, sink.wrong)
    b = max(sink.batches, 1)
    res = dict(devices=devices, senders=n_send, records=total, seconds=t1 - first[0], rate=total / (t1 - first[0]),
               batches=sink.batches, entries=len(sink.table), copy_ms=1e3 * sink.t_copy / b, verify_ms=1e3 * sink.t_verify / b,
               add_ms=1e3 * sink.t_add / b, peer_ms=1e3 * sink.t_peer / b, blocked_s=sink.queue.blocked_s)
    sink.close()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=1 << 23)
    ap.add_argument("--msg", type=int, default=1 << 14, help="records per SENDDP message")
    ap.add_argument("--senders", default="1,4,8")
    ap.add_argument("--one-gpu", default="2,4", help="shard counts to run on GPU 0 alone")
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "server_shards_rate.json"))
    a = ap.parse_args()
    import torch
    from tests.server_util import corrupt, engine_records
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    gpus = torch.cuda.device_count()
    print("card, power limit: %s; %d GPUs visible" % (sr.card(), gpus), flush=True)
    layouts = [list(range(w)) for w in (1, 2, 4, 8) if w <= gpus] + [[0] * int(w) for w in a.one_gpu.split(",") if w]
    recs = engine_records(sr.START, sr.END, sr.KEY, sr.DP, a.records, grid=(132, 128), max_found=1 << 19)[:40 * a.records]
    recs = recs.reshape(-1, 40)
    rng = np.random.default_rng(7)
    wrong = np.sort(rng.choice(a.records, a.records // 20, replace=False))
    recs[wrong] = corrupt(recs.reshape(-1), wrong)
    out = dict(card=sr.card(), gpus=gpus, records=a.records, wrong=len(wrong), msg=a.msg, runs=[], default_capacity={})
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "recs.npy")
        np.save(path, recs)
        for devices in layouts:
            name = ",".join(str(d) for d in devices)
            out["default_capacity"][name] = cap = default_capacity(devices)
            print("--devices %s: default total capacity %d entries (%.2f G)" % (name, cap, cap / 1e9), flush=True)
            for n in [int(v) for v in a.senders.split(",")]:
                r = run(devices, n, path, a.records, len(wrong), a.msg)
                out["runs"].append(r)
                print("  %d senders: %.2f M records/s (%.2f s); per batch (%d): copy %.3f ms, verify+partition %.3f ms, add %.3f ms "
                      "(copies to other GPUs %.3f ms); handlers blocked %.2f s" %
                      (n, r["rate"] / 1e6, r["seconds"], r["batches"], r["copy_ms"], r["verify_ms"], r["add_ms"], r["peer_ms"],
                       r["blocked_s"]), flush=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
