"""End-to-end rate of the DP server (kangaroo_b200.server) on loopback, against the reference's CPU server as the control.

Records: made on the GPU by the engine itself (kgx_convert_dps of a few launches at dp 8 on a 2^100 range, so that no two of
them collide), every one valid; 5 % of them are replaced by wrong copies (one bit of x flipped).  Senders: 1, 4 and 8
processes, each sending its share in SENDDP messages of --msg records over 127.0.0.1.  The server runs in this process
(Server + GpuSink, the code `python -m kangaroo_b200.server` runs), so the script reads when the last record is inserted.
Per sender count it prints records/s inserted end to end (from the first message the server has read to the last record
inserted; the senders' start-up is left out), the ingest thread's time
per batch (host-to-device copy and kgx_resolver_verify_partition at one shard from CUDA events, the add from the host
clock) and how long the handlers blocked on a full queue.  A second pass with 8 senders runs under torch.profiler and gives
the verify kernels' own time per batch: the check, the scans and the partition passes.  The control: the same senders against oracle/_ref/kangaroo_ref_cpu -s (where it was built), its rate read
from its DP Count line, timed from the senders' start (their start-up, about half a second, is inside its window); that server listens on all interfaces while it runs (it has no bind option).  Writes
results/server_rate.json.

    python scripts/server_rate.py [--records 8388608] [--msg 16384]"""
import argparse
import json
import os
import re
import signal
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from kangaroo_b200 import ecmath as ec                                   # noqa: E402

START = 0
END = (1 << 100) - 1
KEY = ec.mul(0x9F3E5C7A1B2D4E6F8091A2B3C4D)
DP = 8
REF_CPU = os.path.join(ROOT, "oracle", "_ref", "kangaroo_ref_cpu")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def sender(port, path, lo, hi, msg):
    """one sender process: records [lo, hi) of the .npy file, in messages of msg records"""
    from tests.server_util import Client
    recs = np.load(path, mmap_mode="r").reshape(-1, 40)
    c = Client(port, timeout=600)
    for o in range(lo, hi, msg):
        while c.send(np.asarray(recs[o:min(o + msg, hi)])) == 2:      # BACKUP: hold the records, poll
            time.sleep(0.2)
    c.close()


def start_senders(n, port, path, total, msg):
    share = (total + n - 1) // n
    return [subprocess.Popen([sys.executable, __file__, "--sender", str(port), path, str(i * share), str(min(total, (i + 1) * share)),
                              str(msg)], cwd=ROOT) for i in range(n)]


def finish(procs, timeout=900):
    try:
        for p in procs:
            p.wait(timeout=timeout)
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
            p.wait()
    return [p.returncode for p in procs]


def run_ours(n_send, path, total, n_wrong, msg):
    from kangaroo_b200.server import GpuSink, Server
    sink = GpuSink(START, END, KEY, DP, capacity=total + (1 << 20), out=lambda s: None)
    srv = Server(START, END, KEY, DP, sink, bind="127.0.0.1", port=0, out=lambda s: None)
    srv.listen()
    first, put = [], sink.put

    def timed_put(m, chunks):                                  # the clock starts at the first message the server has read
        if not first:
            first.append(time.perf_counter())
        put(m, chunks)

    sink.put = timed_put
    try:
        procs = start_senders(n_send, srv.port, path, total, msg)
        while sink.received < total and all(p.poll() in (None, 0) for p in procs) and sink.failed is None:
            time.sleep(0.001)
        t1 = time.perf_counter()
        t0 = first[0]
        rcs = finish(procs)
    finally:
        srv.close()
        sink.finish()
    assert rcs == [0] * n_send and sink.failed is None, (rcs, sink.failed)
    assert sink.received == total and sink.wrong == n_wrong and len(sink.table) <= total - n_wrong, \
        (sink.received, sink.wrong, len(sink.table))
    b = max(sink.batches, 1)
    res = dict(senders=n_send, records=total, seconds=t1 - t0, rate=total / (t1 - t0), batches=sink.batches,
               copy_ms=1e3 * sink.t_copy / b, verify_ms=1e3 * sink.t_verify / b, add_ms=1e3 * sink.t_add / b,
               blocked_s=sink.queue.blocked_s)
    sink.close()
    return res


def profiled_verify(path, total, n_wrong, msg, outdir):
    """8 senders under torch.profiler -> the verify kernels' device time per batch (check, scan, partition)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        r = run_ours(8, path, total, n_wrong, msg)
    prof.export_chrome_trace(os.path.join(outdir, "server_rate.pt.trace.json"))
    us = {"check": 0.0, "scan": 0.0, "partition": 0.0}
    for e in prof.key_averages():
        name = e.key
        t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
        if "wt_check_entries_kernel" in name and "Dp40Check" in name:
            us["check"] += t
        elif "k_counts" in name or (("k_hist" in name or "k_scatter" in name) and "Verified" in name):
            us["partition"] += t
        elif "DeviceScan" in name or "ScanKernel" in name or "DeviceScanInitKernel" in name:
            us["scan"] += t                                    # cub's scan (the device table's own scans count here too)
    return {k: v / 1e3 / max(r["batches"], 1) for k, v in us.items()}, r


def run_ref(n_send, path, total, msg, tmpdir):
    """the reference CPU server with the same senders -> records/s from its DP Count line, or None when it is not built"""
    if not os.path.exists(REF_CPU):
        return None
    from tests.ranks_util import free_port
    cfg = os.path.join(tmpdir, "ref.txt")
    with open(cfg, "w") as f:
        f.write("%X\n%X\n04%064X%064X\n" % (START, END, KEY[0], KEY[1]))
    port = free_port()
    log = open(os.path.join(tmpdir, "ref_server.log"), "w+")
    unbuf = ["stdbuf", "-o0"] if subprocess.run(["which", "stdbuf"], capture_output=True).returncode == 0 else []
    p = subprocess.Popen(unbuf + [REF_CPU, "-s", "-d", str(DP), "-sp", str(port), cfg], stdout=log, stderr=subprocess.STDOUT, cwd=tmpdir)
    try:
        deadline = time.monotonic() + 60
        while "listening" not in open(log.name).read() and time.monotonic() < deadline:
            time.sleep(0.1)
        t0 = time.perf_counter()
        procs = start_senders(n_send, port, path, total, msg)
        finish(procs)
        count, t1 = 0.0, None
        deadline = time.monotonic() + 600
        while time.monotonic() < deadline:
            m = re.findall(r"DP Count 2\^([0-9.]+)", open(log.name).read())
            if m and 2 ** float(m[-1]) >= total * 0.99:
                count, t1 = 2 ** float(m[-1]), time.perf_counter()
                break
            time.sleep(0.05)
    finally:
        p.send_signal(signal.SIGINT)
        try:
            p.wait(timeout=10)
        except subprocess.TimeoutExpired:
            p.kill()
            p.wait()
    if t1 is None:
        return dict(senders=n_send, rate=None)
    return dict(senders=n_send, records=count, seconds=t1 - t0, rate=count / (t1 - t0))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=1 << 23)
    ap.add_argument("--msg", type=int, default=1 << 14, help="records per SENDDP message")
    ap.add_argument("--senders", default="1,4,8")
    ap.add_argument("--no-ref", action="store_true")
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "server_rate.json"))
    ap.add_argument("--sender", nargs=5, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.sender:
        port, path, lo, hi, msg = a.sender
        sender(int(port), path, int(lo), int(hi), int(msg))
        return
    from tests.server_util import corrupt, engine_records
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    print("card, power limit: %s" % card(), flush=True)
    recs = engine_records(START, END, KEY, DP, a.records, grid=(132, 128), max_found=1 << 19)[:40 * a.records].reshape(-1, 40)
    rng = np.random.default_rng(7)
    wrong = np.sort(rng.choice(a.records, a.records // 20, replace=False))
    recs[wrong] = corrupt(recs.reshape(-1), wrong)
    out = dict(card=card(), records=a.records, wrong=len(wrong), msg=a.msg, bytes_per_record=40, bytes_per_message=25, ours=[], ref=[])
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "recs.npy")
        np.save(path, recs)
        for n in [int(v) for v in a.senders.split(",")]:
            r = run_ours(n, path, a.records, len(wrong), a.msg)
            out["ours"].append(r)
            print("ours  %d senders: %.2f M records/s (%.2f s); per batch (%d): copy %.3f ms, verify %.3f ms, add %.3f ms; handlers "
                  "blocked %.2f s" % (n, r["rate"] / 1e6, r["seconds"], r["batches"], r["copy_ms"], r["verify_ms"], r["add_ms"],
                                      r["blocked_s"]), flush=True)
        kern, r = profiled_verify(path, a.records, len(wrong), a.msg, os.path.dirname(a.out))
        out["verify_kernels_ms_per_batch"] = kern
        print("profiled (8 senders, %d batches): check %.3f ms, scan %.3f ms, partition %.3f ms per batch" %
              (r["batches"], kern["check"], kern["scan"], kern["partition"]), flush=True)
        if not a.no_ref:
            for n in [int(v) for v in a.senders.split(",")]:
                r = run_ref(n, path, a.records, a.msg, tmp)
                out["ref"].append(r)
                if r is None:
                    print("ref   %d senders: not measured (oracle/_ref/kangaroo_ref_cpu not built)" % n, flush=True)
                elif r["rate"] is None:
                    print("ref   %d senders: not measured (its DP Count did not reach the records sent)" % n, flush=True)
                else:
                    print("ref   %d senders: %.2f M records/s (%.2f s)" % (n, r["rate"] / 1e6, r["seconds"]), flush=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
