#!/usr/bin/env python
"""bench.py -- MJump/s of the H100 kangaroo jump engine (BASELINE.json metric) + roofline + CPU baseline.

One "step" = one GPUEngine::Launch on the full herd: NB_RUN=64 jumps for every kangaroo of the default
grid (2*SMs x 128 threads x 128; on an H100 SXM 2*132 x 128 x 128 = 4,325,376 kangaroos, the size the reference's
GetGridSize picks, GPUEngine.cu:301-303), jump table of the in80 configuration (VC_CUDA8/in80.txt: 2^79.8 range -> rangePower 80,
dp = 16), the reference's own throughput accounting `nbKangaroo * NB_RUN` per Launch (Kangaroo.cpp:575).

  value : jumps / device time of exactly K launches (state resident in HBM, DP slabs left on the device)
  e2e   : the same K launches through the reference-shaped host API (GPUEngine.Launch -> std::vector<ITEM>
          equivalent): every step waits for the kernel, reads the DP records back to HOST memory and decodes
          them, exactly what Kangaroo::SolveKeyGPU consumes.  The herd itself is resident by design of the
          reference interface (SetKangaroos once, GPUEngine.cu:381-433), so h2d per step is 0 payload bytes.
  roofline : integer-multiply bound (SURVEY.md 8d): 416 IMAD.WIDE per jump (5 ModMult x 74 + ModSqr x 46) against
          the wide-IMAD issue rate measured in the same run (kgx_bench_raw), plus the HBM view.
  cpu_baseline : the reference's SolveKeyCPU inner loop (oracle/_ref/libkref.so = unmodified SECPK1 code) on all
          host cores for a bounded sample.

`--impl reference` times that CPU implementation alone.  Under torchrun (N>1) one rank per GPU, independent
herds (weak scaling), DP records gathered to rank 0 over NCCL every step.
`--dump-outputs DIR` writes what the last timed step computed (see dump_outputs) so two builds can be compared.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
# stdout carries exactly one JSON line (rank 0): whatever NCCL logs (NCCL_DEBUG=VERSION/WARN/INFO) goes to stderr
os.environ.setdefault("NCCL_DEBUG_FILE", "/dev/stderr")

NB_RUN = 64
ALGO_IMAD_PER_JUMP = 416          # SURVEY.md 8d / BASELINE.md 3
ALGO_BYTES_PER_JUMP = 2.5         # 2 x 80 B per kangaroo per 64 jumps
DESIGN_BYTES_PER_JUMP = {"stream": 224.0, "resident": 2.5}   # DESIGN.md 3.1 / 3.2


def host_cores():
    try:
        return len(os.sched_getaffinity(0))
    except Exception:
        return os.cpu_count() or 1


_CPU_THREADS = None
CALIB_PATH = os.path.join(tempfile.gettempdir(), "kgx_cpu_calibration.json")   # never inside the (possibly read-only) tree


def cpu_threads(be):
    """Thread count of the CPU arm, calibrated ONCE per host and shared by `--impl reference`, the cpu_baseline leg and the
    product-level run, so that all three use the same count.  The visible CPU count can exceed what the container may run
    (cgroup quota), so the candidate with the best short-run rate is kept and cached in the temporary directory, keyed by
    host name and visible core count."""
    global _CPU_THREADS
    if _CPU_THREADS is not None:
        return _CPU_THREADS
    import socket
    key = "%s/%d" % (socket.gethostname(), host_cores())
    try:
        cache = json.load(open(CALIB_PATH))
        if cache.get("key") == key:
            _CPU_THREADS = int(cache["threads"])
            return _CPU_THREADS
    except Exception:
        pass
    avail = host_cores()
    cands = sorted({c for c in (avail, avail // 2, avail // 4, 32, 16, 8) if 1 <= c <= avail})
    best, rates = (0.0, 1), {}
    for c in cands:
        r = 0.0
        for _ in range(2):                                      # best of two short runs per candidate
            j, sec = be.bench_cpu(c, 160, 80)
            r = max(r, j / sec)
        rates[c] = r / 1e6
        if r > best[0]:
            best = (r, c)
    _CPU_THREADS = best[1]
    try:
        json.dump({"key": key, "threads": _CPU_THREADS, "mjump_s_by_threads": rates}, open(CALIB_PATH, "w"))
    except Exception:
        pass
    return _CPU_THREADS


def cpu_reference_run(seconds_target):
    """SolveKeyCPU inner loop through the reference's own Int/IntGroup code on all the host threads it can use."""
    from oracle import kgo
    if os.path.exists(kgo.Reference.path):
        be, kind = kgo.Reference(), "reference"
    else:
        be, kind = kgo.Oracle(), "port"
    cores = cpu_threads(be)
    jumps, sec = be.bench_cpu(cores, 256, 80)                       # rate probe: 256 jumps x 1024 kangaroos / thread
    rate = jumps / sec
    per_thread = max(256, int(seconds_target * rate / cores / 1024))
    jumps, sec = be.bench_cpu(cores, per_thread, 80)
    return dict(value=jumps / sec / 1e6, unit="MJump/s", cores=cores, kind=kind,
                sample="%d threads x 1024 kangaroos x %d jumps (SolveKeyCPU inner loop, CPU_GRP_SIZE=1024, rangePower 80), %.1f s"
                       % (cores, per_thread, sec)), sec


def cpu_product_run(threads, seconds=20.0):
    """SURVEY 8(d) item 1: the reference PROGRAM itself (oracle/_ref/kangaroo_ref_cpu = unmodified main/Kangaroo/HashTable/SECPK1,
    CPU build) with -t <threads> on the 64-bit fixture for a fixed time; rate = growth of its own `Count 2^x` between two status
    lines stamped on arrival (its displayed average has an accumulation bug, Thread.cpp:294-300)."""
    import re
    import select
    exe = os.path.join(ROOT, "oracle", "_ref", "kangaroo_ref_cpu")
    cfg = os.path.join(ROOT, "tests", "golden", "puzzle110_window80.txt")       # cannot finish in 20 s: steady state only
    if not os.path.exists(exe):
        return None
    p = subprocess.Popen([exe, "-t", str(threads), "-d", "20", cfg], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL)
    t_end, buf, marks = time.time() + seconds + 6.0, b"", []
    try:
        while time.time() < t_end:
            r, _, _ = select.select([p.stdout], [], [], 0.5)
            if not r:
                continue
            chunk = os.read(p.stdout.fileno(), 65536)
            if not chunk:
                break
            buf += chunk
            ms = re.findall(rb"Count 2\^([0-9.]+)", buf)
            if ms and (not marks or marks[-1][1] != ms[-1]):
                marks.append((time.time(), ms[-1]))
            buf = buf[-4096:]
    finally:
        p.kill()
        p.wait()
    if len(marks) < 3:
        return None
    (ta, ca), (tb, cb) = marks[1], marks[-1]                       # skip the first line (thread start-up)
    rate = (2.0 ** float(cb) - 2.0 ** float(ca)) / max(tb - ta, 1e-9)
    return dict(value=rate / 1e6, unit="MJump/s", cores=threads, kind="reference-program",
                sample="kangaroo (reference, CPU build) -t %d on a 2^80 window for %.0f s: Count 2^%s -> 2^%s"
                       % (threads, tb - ta, ca.decode(), cb.decode()))


class ClockSampler(threading.Thread):
    """One long-lived `nvidia-smi -lms 50` (read-only queries) whose lines are stamped on arrival; result() keeps the
    samples that fell inside the timed regions."""
    Q = "clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown," \
        "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"
    NAMES = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]

    def __init__(self, dev):
        super().__init__(daemon=True)
        self.dev, self.rows, self.stop_flag, self.windows, self.proc = dev, [], False, [], None

    def run(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.dev), "--query-gpu=" + self.Q, "--format=csv,noheader,nounits",
                                          "-lms", "50"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            for line in self.proc.stdout:
                self.rows.append((time.perf_counter(), line.strip().split(",")))
                if self.stop_flag:
                    break
        except Exception:
            pass

    def window(self, t0, t1):
        self.windows.append((t0, t1))

    def stop(self):
        self.stop_flag = True
        if self.proc is not None:
            try:
                self.proc.terminate()
            except Exception:
                pass
        self.join(timeout=2)

    def result(self):
        mhz, reasons, max_mhz = [], set(), None
        for t, f in self.rows:
            try:
                inside = any(a <= t <= b for a, b in self.windows)
                max_mhz = float(f[1])
                if inside:
                    mhz.append(float(f[0]))
                    for n, v in zip(self.NAMES, f[2:]):
                        if "Active" in v and "Not" not in v:
                            reasons.add(n)
            except Exception:
                continue
        mhz.sort()
        return dict(sm_mhz=(mhz[len(mhz) // 2] if mhz else None), sm_max_mhz=max_mhz, reasons=sorted(reasons), samples=len(mhz))


def load_in80_table():
    """Jump table for rangePower 80 from the reference-generated fixture (tests/golden/jump_golden.json)."""
    from tests.golden_util import load_cases
    for c in load_cases():
        if c["range_power"] == 80:
            return c
    raise RuntimeError("in80 fixture missing")


def build_herd(eng, case, rank):
    """Synthetic herd shaped like Kangaroo::CreateHerd (Kangaroo.cpp:670-738): every kangaroo gets its own uniform
    random distance in the 2^80 range (numpy PCG64, seeded per rank), wild ones shifted by -width/2 (mod n) and started
    at key + d*G.  The point arithmetic runs on the device (kgx_create_herd), so all walkers are distinct valid
    curve points; no part of the oracle is involved."""
    import numpy as np
    from kangaroo_b200 import random_herd_arrays
    rng = np.random.Generator(np.random.PCG64(1234 + rank))
    wdiv2 = case["width_div2"]
    eng.SetWildOffset(wdiv2)
    sc, d128 = random_herd_arrays(eng.nbKangaroo, 80, wdiv2, rng)
    eng.CreateHerdRaw(sc, d128, case["key"])
    return sc


def _limb_rows(vals, limbs):
    import numpy as np
    out = np.zeros((len(vals), limbs), dtype=np.uint64)
    for i, v in enumerate(vals):
        for k in range(limbs):
            out[i, k] = (int(v) >> (64 * k)) & 0xFFFFFFFFFFFFFFFF
    return out


def shim_prepare(eng, case, sc, local_rank):
    """Dump what the C++ harness uploads through SetParams/SetKangaroos: the jump table and the freshly created herd (positions
    read back from the device, true distances mod n) -- called BEFORE any launch so that (x, y, d) are consistent."""
    import tempfile
    import numpy as np
    if not os.path.exists(os.path.join(ROOT, "build", "kgx_shim_bench")):
        return None
    ax, ay, _ = eng.GetKangaroosRaw()
    tmp = tempfile.mkdtemp(prefix="kgx_shim_%d_" % local_rank)
    tab_path, herd_path = os.path.join(tmp, "table.bin"), os.path.join(tmp, "herd.bin")
    jd, jpx, jpy = case["table"]
    as_rows = lambda a, limbs: (np.ascontiguousarray(a, dtype=np.uint64)[:, :limbs] if isinstance(a, np.ndarray) else _limb_rows(a, limbs))
    tab = np.concatenate([as_rows(jd, 2), as_rows(jpx, 4), as_rows(jpy, 4)], axis=1)                 # 32 x 10
    with open(tab_path, "wb") as f:
        f.write(tab.tobytes()); f.write(_limb_rows([case["width_div2"]], 4).tobytes())
    np.concatenate([ax, ay, np.ascontiguousarray(sc, dtype=np.uint64)], axis=1).tofile(herd_path)   # n x 12
    return tmp, tab_path, herd_path


def shim_run(prep, gx, gy, local_rank, dp, warmup, steps):
    """Headline e2e leg: K steps through the reference's C++ interface -- build/kgx_shim_bench constructs `class GPUEngine`
    (reference header, GPUEngine_b200.cpp shim), SetKangaroos(Int*...) from host arrays, callKernel, K x Launch(std::vector<ITEM>&)
    with the per-record Int marshalling and ModSubK1order of the reference's Launch (GPUEngine.cu:653-675).
    -> (seconds for K steps, DP items returned, upload seconds)"""
    tmp, tab_path, herd_path = prep
    exe = os.path.join(ROOT, "build", "kgx_shim_bench")
    try:
        p = subprocess.run([exe, str(local_rank), str(gx), str(gy), str(dp), str(warmup), str(steps), tab_path, herd_path],
                           capture_output=True, text=True, timeout=900)
        line = [ln for ln in p.stdout.splitlines() if ln.startswith("{")]
        if p.returncode != 0 or not line:
            raise RuntimeError("kgx_shim_bench failed: " + (p.stdout + p.stderr)[-500:])
        r = json.loads(line[-1])
        shim_run.last = r
        return r["seconds"], r["items"], r["upload_s"]
    finally:
        for f in (tab_path, herd_path):
            try:
                os.remove(f)
            except OSError:
                pass
        try:
            os.rmdir(tmp)
        except OSError:
            pass


def _limbs32(a):
    """(n, k) uint64 limbs -> (n, 2k) float64 of 32-bit limbs, little-endian: exact in float64."""
    import numpy as np
    return np.ascontiguousarray(a, dtype=np.uint64).view(np.uint32).astype(np.float64)


def dump_outputs(out_dir, eng, lib, max_found, sample=65536, seed=0):
    """What the last timed launch computed, as a caller of the device-resident path receives it: the DP records of that
    launch (sorted by kangaroo index, then x: their order in the slab depends on thread timing) and the herd state it
    leaves behind, for a fixed seeded sample of kangaroos.  Every array is float64 (256-bit values as 32-bit limbs)."""
    import ctypes
    import numpy as np
    from kangaroo_b200._lib import Item
    os.makedirs(out_dir, exist_ok=True)
    items = (Item * max_found)()
    nI, nF = ctypes.c_uint32(0), ctypes.c_uint32(0)
    rc = lib.kgx_collect(eng._h, items, max_found, ctypes.byref(nI), ctypes.byref(nF), 0, 0)   # no relaunch: read the slab
    assert rc == 0, lib.kgx_last_error(eng._h)
    raw = np.frombuffer(items, dtype=np.uint64, count=int(nI.value) * 7).reshape(-1, 7)
    words = raw.view(np.uint32)                                       # x: words 0..7, d: 8..11, kidx: 12..13
    order = np.lexsort(tuple(words[:, w] for w in range(7, -1, -1)) + (raw[:, 6],))
    raw = raw[order]
    ax, ay, ad = eng.GetKangaroosRaw()
    rng = np.random.Generator(np.random.PCG64(seed))
    idx = np.sort(rng.choice(ax.shape[0], size=min(sample, ax.shape[0]), replace=False))
    arrays = {"dp_count": np.array([nF.value], dtype=np.float64), "dp_x": _limbs32(raw[:, 0:4]), "dp_d": _limbs32(raw[:, 4:6]),
              "dp_kidx": raw[:, 6].astype(np.float64), "state_index": idx.astype(np.float64),
              "state_x": _limbs32(ax[idx]), "state_y": _limbs32(ay[idx]), "state_d": _limbs32(ad[idx])}
    for name, a in arrays.items():
        np.save(os.path.join(out_dir, name + ".npy"), a)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--grid", default="", help="x,y override (default 2*SMs,128)")
    ap.add_argument("--dp", type=int, default=16)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--dump-outputs", default="", metavar="DIR",
                    help="write the DP records and a sampled herd state of the last timed step as DIR/<name>.npy (rank 0)")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")

    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    steps, warmup = args.steps, max(args.warmup, 0)

    if args.impl == "reference":
        if rank != 0:
            return 0
        per_step_s = max(0.5, min(4.0, 100.0 / max(steps, 1)))     # bounded sample: the K timed steps end within ~2 min
        base, _ = cpu_reference_run(per_step_s)
        vals = []
        for _ in range(warmup):
            cpu_reference_run(min(1.0, per_step_s))
        for _ in range(steps):
            r, _ = cpu_reference_run(per_step_s)
            vals.append(r["value"])
        v = sum(vals) / len(vals)
        base["value"] = v
        print(json.dumps(dict(impl="reference", metric="MJump/s (kangaroo jumps/sec)", value=v, unit="MJump/s", n_gpus=args.gpus,
                              steps=len(vals), warmup=warmup, ms_per_step=per_step_s * 1e3, higher_is_better=True, scaling="weak",
                              vs_baseline=None, dtype="u32x8 (256-bit modular integer)", data="synthetic",
                              config={"workload": "in80.txt: rangePower 80 jump table; reference SolveKeyCPU inner loop (Kangaroo.cpp:375-433) on the "
                                                  "host cores, CPU_GRP_SIZE=1024 kangaroos per thread, bounded sample per step",
                                      "group": 1024}, cpu_baseline=base,
                              e2e=dict(value=v, unit="MJump/s", h2d_bytes_per_step=0, d2h_bytes_per_step=0))))
        return 0

    import numpy as np
    import torch
    import kangaroo_b200
    from kangaroo_b200 import GPUEngine

    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device -- the jump engine has no CPU fallback")
    torch.cuda.set_device(local_rank)
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))

    gx, gy = (int(v) for v in args.grid.split(",")) if args.grid else GPUEngine.GetGridSize(local_rank, 0, 0)
    case = load_in80_table()
    max_found = 1 << 17                                            # Kangaroo.cpp:523 (65536*2)
    eng = GPUEngine(gx, gy, local_rank, max_found)
    n = eng.nbKangaroo
    dp_mask = (~((1 << (64 - args.dp)) - 1)) & 0xFFFFFFFFFFFFFFFF if args.dp else 0
    eng.SetParams(dp_mask, *case["table"])
    herd_scalars = build_herd(eng, case, rank)
    try:
        shim_prep = shim_prepare(eng, case, herd_scalars, local_rank)
    except OSError as exc:                                         # e.g. no room for the ~0.4 GB herd file: keep the C-ABI e2e leg
        print("bench.py: C++ shim leg skipped on rank %d: %s" % (rank, exc), file=sys.stderr)
        shim_prep = None
    del herd_scalars

    from kangaroo_b200.dist import DPGather
    gather = DPGather(eng, dist, rank, world, torch) if world > 1 else None

    def barrier():
        torch.cuda.synchronize()
        if dist is not None:
            dist.barrier()
        torch.cuda.synchronize()

    # ---- device-resident leg: K launches, DP slabs stay on the device -----------------------------------
    lib = kangaroo_b200.load_library()
    import ctypes
    nI, nF = ctypes.c_uint32(0), ctypes.c_uint32(0)

    def device_step():
        # wait for the launch in flight, start the next one; cap=0 -> no host readback of records
        rc = lib.kgx_collect(eng._h, eng._items, 0, ctypes.byref(nI), ctypes.byref(nF), 0, 1)
        assert rc == 0, lib.kgx_last_error(eng._h)
        if gather is not None:
            gather.step(int(nF.value))
        return eng.last_launch_ms(), int(nF.value)

    eng.callKernel()
    for _ in range(max(warmup, 3)):
        device_step()
    sampler = ClockSampler(local_rank); sampler.start()
    launches0 = eng.kernel_launches()
    barrier()
    t0 = time.perf_counter()
    kernel_ms, found = [], 0
    for _ in range(steps):
        ms, nf = device_step()
        kernel_ms.append(ms); found += nf
    eng.sync()
    barrier()
    wall = time.perf_counter() - t0
    sampler.window(t0, t0 + wall)
    gpu_launches = eng.kernel_launches() - launches0
    # the K timed launches are exactly the K kernels completed inside the region: (K-1) collected + the one synced
    kernel_ms = kernel_ms[1:] + [eng.last_launch_ms()]
    dev_s = sum(kernel_ms) / 1e3
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, eng, lib, max_found)

    # ---- end-to-end leg through the C ABI with HOST buffers: kgx_collect(..., relaunch=1) is exactly the body of
    # GPUEngine::Launch (GPUEngine.cu:607-679): wait for the kernel, start the next one, copy this launch's DP records
    # device -> pinned staging -> the caller's host array of 56-byte items (what SolveKeyGPU then hashes).
    from kangaroo_b200._lib import Item
    host_items = (Item * max_found)()
    eng.callKernel()

    def e2e_step():
        rc = lib.kgx_collect(eng._h, host_items, max_found, ctypes.byref(nI), ctypes.byref(nF), 0, 1)
        assert rc == 0, lib.kgx_last_error(eng._h)
        if gather is not None:
            gather.step(int(nF.value))
        return int(nI.value)

    for _ in range(2):
        e2e_step()
    barrier()
    t1 = time.perf_counter()
    d2h = 0
    for _ in range(steps):
        d2h += 4 + e2e_step() * 56
    eng.sync()
    barrier()
    e2e_s = time.perf_counter() - t1
    sampler.window(t1, t1 + e2e_s)

    # ---- headline e2e leg: the same K steps through the reference's own C++ class interface (GPUEngine_b200.cpp shim), one
    # harness process per rank on its GPU (the reference runs one GPUEngine per host thread, Kangaroo.cpp:1041-1047)
    shim_s, shim_items, shim_upload = 0.0, 0, 0.0
    if shim_prep is not None:
        barrier()
        t3 = time.perf_counter()
        shim_s, shim_items, shim_upload = shim_run(shim_prep, gx, gy, local_rank, args.dp, max(warmup, 3), steps)
        sampler.window(t3 + shim_upload, time.perf_counter())
        barrier()
    sampler.stop()

    # ---- worst case for context: the whole herd round-trips through HOST memory every step (not how the reference
    # interface is used -- SetKangaroos is a one-time upload -- but it bounds what a host-resident caller would see)
    rt_steps, rt_s, rt_h2d, rt_d2h = 0, 0.0, 0, 0
    if world == 1:
        ax, ay, ad = eng.GetKangaroosRaw()
        eng.sync()
        t2 = time.perf_counter()
        for _ in range(2):
            eng.SetKangaroosRaw(ax, ay, ad)
            eng.callKernel()
            items = eng.Launch(relaunch=False)
            ax, ay, ad = eng.GetKangaroosRaw()
            rt_steps += 1; rt_h2d += n * 80; rt_d2h += n * 80 + 4 + len(items) * 56
        rt_s = time.perf_counter() - t2

    own_kernel_value = float(n) * NB_RUN * steps / dev_s / 1e6        # this rank alone, before the max over ranks
    t = torch.tensor([dev_s, wall, e2e_s, shim_s], dtype=torch.float64, device="cuda")
    if dist is not None:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    dev_s, wall, e2e_s, shim_s = (float(v) for v in t.tolist())
    total_jumps = float(n) * NB_RUN * steps * world
    value = total_jumps / wall / 1e6                 # whole job, wall clock between barriers (max over ranks)
    kernel_value = float(n) * NB_RUN * steps / dev_s / 1e6
    # one line per rank on stderr (the JSON line on stdout stays rank 0's alone): device, NCCL, this rank's own rates
    nccl_v = ".".join(str(v) for v in torch.cuda.nccl.version()) if world > 1 else "-"
    print("[bench rank %d/%d] cuda:%d %s | NCCL %s | kernel %.1f MJump/s | %d DPs/step | gathered to rank 0: %s"
          % (rank, world, local_rank, torch.cuda.get_device_name(local_rank), nccl_v, own_kernel_value, found // max(steps, 1),
             "yes" if gather is not None else "n/a (single GPU)") + "\n", file=sys.stderr, end="", flush=True)
    cabi_value = total_jumps / e2e_s / 1e6
    e2e_value = total_jumps / shim_s / 1e6 if shim_s > 0 else cabi_value

    if rank == 0:
        clocks = sampler.result()
        mhz = clocks["sm_mhz"] or clocks["sm_max_mhz"] or 1980.0    # 1980 MHz: H100 SXM maximum SM clock
        sms = torch.cuda.get_device_properties(local_rank).multi_processor_count
        # multiplier roofline: IMAD.WIDE.U32 issue rate measured NOW on this GPU (kgx_bench_raw kind 0, best of 3)
        imad_peak = 0.0
        for _ in range(3):
            ms_, ops_ = ctypes.c_float(0), ctypes.c_double(0)
            assert lib.kgx_bench_raw(local_rank, 0, 20000, ctypes.byref(ms_), ctypes.byref(ops_)) == 0
            imad_peak = max(imad_peak, ops_.value / (ms_.value * 1e-3))
        # second measured view: what the multiplier pipe sustains inside real carry chains (kgx_bench_raw kind 1: dependent fe_mul
        # chains, 73 wide IMAD each) -- it can run above the accumulate-probe, so the larger of the two is the measured peak
        chain_peak = 0.0
        for _ in range(2):
            ms_, ops_ = ctypes.c_float(0), ctypes.c_double(0)
            assert lib.kgx_bench_raw(local_rank, 1, 2000, ctypes.byref(ms_), ctypes.byref(ops_)) == 0
            chain_peak = max(chain_peak, 73.0 * ops_.value / (ms_.value * 1e-3))
        probe_peak = imad_peak
        imad_peak = max(imad_peak, chain_peak)
        nominal_peak = sms * 32.0 * mhz * 1e6          # quarter-rate pipe: 32 lane-ops/clk/SM at the SM clock seen during the run
        achieved = kernel_value * 1e6 * ALGO_IMAD_PER_JUMP
        mode = eng.kernel
        hbm_peak, hbm_src = 3350.0, "H100 SXM data sheet (HBM3)"
        l2_mb = torch.cuda.get_device_properties(local_rank).L2_cache_size / 2**20
        hbm_ach = kernel_value * 1e6 * ALGO_BYTES_PER_JUMP / 1e9
        out = dict(
            metric="MJump/s (kangaroo jumps/sec)", value=value, unit="MJump/s", n_gpus=world, steps=steps, warmup=max(warmup, 3),
            ms_per_step=wall / steps * 1e3, higher_is_better=True, scaling="weak", vs_baseline=None,
            dtype="u32x8 (256-bit modular integer)", data="synthetic",
            config={"workload": "in80.txt: rangePower 80 jump table, dp=%d, grid %dx%d -> %d kangaroos/GPU x NB_RUN=64 jumps per step"
                                % (args.dp, gx, gy, n),
                    "state_bytes_per_gpu": n * 80,
                    "l2_note": "%.0f MB of kangaroo state per GPU > %.0f MB L2; every step streams all of it" % (n * 80 / 1e6, l2_mb),
                    "dp_found_per_step": found / max(steps, 1)},
            kernel_only={"value": kernel_value, "unit": "MJump/s/GPU", "ms_per_launch": dev_s / steps * 1e3,
                         "how": "CUDA events on the engine stream around each jump_kernel launch"},
            e2e={"value": e2e_value, "unit": "MJump/s", "h2d_bytes_per_step": 0,
                 "d2h_bytes_per_step": (4 + shim_items * 56.0 / max(steps, 1)) if shim_s > 0 else d2h / max(steps, 1),
                 "how": ("build/kgx_shim_bench: the reference's own `class GPUEngine` (unchanged header, GPUEngine_b200.cpp over libkgx.so): "
                         "SetKangaroos(Int*) once, then K x Launch(std::vector<ITEM>&) = wait, relaunch, DP records device -> host -> Int "
                         "marshalling + ModSubK1order per record (GPUEngine.cu:607-679); host-clock around the K calls, max over ranks"
                         if shim_s > 0 else
                         "kgx_collect(relaunch=1) loop through the C ABI with host item buffers (C++ harness not built)"),
                 "one_time_upload_s": shim_upload,
                 "get_kangaroos_s": getattr(shim_run, "last", {}).get("get_kangaroos_s")},
            e2e_c_abi={"value": cabi_value, "unit": "MJump/s", "d2h_bytes_per_step": d2h / max(steps, 1),
                       "how": "kgx_collect(relaunch=1) from Python/ctypes into a host array of 56-byte items: the C ABI alone, no Int marshalling"},
            roofline={"bound": "imad", "achieved": achieved / 1e12, "peak": imad_peak / 1e12, "unit": "TIMAD/s (32x32->64 multiply-adds)",
                      "frac": achieved / imad_peak,
                      "algorithmic_imad_per_jump": ALGO_IMAD_PER_JUMP,
                      "peak_how": "best of two live measurements of the wide-multiply pipe on this GPU: independent IMAD.WIDE accumulate probe "
                                  "(kgx_bench_raw kind 0: %.2f T/s = %.1f lane-ops/clk/SM) and 73 x the dependent fe_mul-chain rate (kind 1: %.2f T/s "
                                  "= %.1f lane-ops/clk/SM) at %.0f MHz on %d SMs.  Whether this pipe or HBM (hbm.designed_frac) bounds the kernel is not "
                                  "measured: no DRAM byte counter is read"
                                  % (probe_peak / 1e12, probe_peak / sms / (mhz * 1e6), chain_peak / 1e12, chain_peak / sms / (mhz * 1e6), mhz, sms),
                      "nominal": {"peak": nominal_peak / 1e12, "frac": achieved / nominal_peak,
                                  "how": "32 lane-ops/clk/SM (quarter-rate pipe) x %d SMs x %.0f MHz -- never reached by any probe" % (sms, mhz)},
                      "hbm": {"bound": "hbm", "achieved": hbm_ach, "peak": hbm_peak, "unit": "GB/s", "frac": hbm_ach / hbm_peak,
                              "peak_source": hbm_src, "algorithmic_bytes_per_jump": ALGO_BYTES_PER_JUMP,
                              "designed_bytes_per_jump": DESIGN_BYTES_PER_JUMP.get(mode),
                              "designed_gbs": kernel_value * 1e6 * DESIGN_BYTES_PER_JUMP.get(mode, 0) / 1e9,
                              "designed_frac": kernel_value * 1e6 * DESIGN_BYTES_PER_JUMP.get(mode, 0) / 1e9 / hbm_peak}},
            kernel_mode=mode,
            gpu_launches=int(gpu_launches), clocks=clocks)
        if rt_steps:
            out["e2e_state_roundtrip"] = {"value": float(n) * NB_RUN * rt_steps / rt_s / 1e6, "unit": "MJump/s",
                                          "h2d_bytes_per_step": rt_h2d / rt_steps, "d2h_bytes_per_step": rt_d2h / rt_steps,
                                          "how": "SetKangaroos (pageable host -> device) + Launch + GetKangaroos every step"}
        if not args.no_cpu_baseline and world >= 1:
            base, _ = cpu_reference_run(12.0)
            out["cpu_baseline"] = base
            out["speedup_vs_cpu_e2e"] = e2e_value / base["value"]
            if world == 1:
                prod = cpu_product_run(base["cores"], 20.0)       # SURVEY 8(d) item 1: the reference program itself, same thread count
                if prod is not None:
                    out["cpu_baseline_product"] = prod
        print(json.dumps(out))
    eng.close()
    if dist is not None:
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
