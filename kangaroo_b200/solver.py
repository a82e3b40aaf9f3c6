"""Stand-alone multi-GPU driver of the jump engine: the role Kangaroo::Run / SolveKeyGPU (Kangaroo.cpp:913-1083,
510-644) plays in the reference, with the reference's TCP client/server (Network.cpp) replaced in-box by one process
per GPU and an NCCL gather of the DP records to rank 0 (kangaroo_b200/dist.py).  Kept deliberately small: it exists to
exercise the engine end to end (BASELINE config 4) -- the full-featured caller remains the reference's own program
linked against the engine (INTEGRATION.md).

Per step (= one GPUEngine::Launch on every rank) nothing on the data path is Python:
  engine      kgx_collect(cap=0, relaunch=1): wait for launch i, start launch i+1, no host copy of records
  device      kgx_convert_dps: HashTable::Convert of launch i's DPs -> 40-byte `DP` records (Kangaroo.h:94-101)
  NCCL        all_gather(count) + gather(records) to rank 0          (dist.DPGather, wire "dp40")
  rank 0      one D2H copy -> (ingest thread, one step behind, overlapping the next launch) kgi_add: the reference's HashTable,
              bucket-sharded multi-threaded insert (ingest.DPTable)
              -> events: KGI_EV_COLLISION -> kgi_resolve (CollisionCheck/CheckKey with the reference's Secp256K1)
                         KGI_EV_RESET     -> (rank, kIdx) sent back to the owner, which re-creates that kangaroo
                                             (Kangaroo.cpp:601-609: CreateHerd(1) + SetKangaroo)
  all ranks   one small broadcast: [stop, n_resets, (rank, kIdx) ...]

  single GPU :  python -m kangaroo_b200.solver in.txt --dp 12
  N GPUs     :  torchrun --nproc-per-node N -m kangaroo_b200.solver in.txt --dp 12
"""
import argparse
import ctypes
import os
import queue
import sys
import threading
import time

import numpy as np

from . import ecmath as ec
from .engine import GPUEngine, NB_JUMP, NB_RUN, WILD, random_herd_arrays
from .dist import DPGather, SlabView, DP40_BYTES
from .ingest import DPTable, EV_RESET, EV_COLLISION

ORDER = ec.N
MAX_RESETS = 255          # per step, carried in the control broadcast


def create_jump_table(range_power):
    """Kangaroo::CreateJumpTable (Kangaroo.cpp:742-832, non-symmetry): 32 distances of rangePower/2+1 bits from MT19937
    seeded 0x600DCAFE (constant "for compatibility of workfiles"), redrawn until the mean is within 2^(jumpBit-1.05 ..
    -0.95); points = d*G.  numpy's RandomState is the same MT19937 with the same seeding, Int::Rand(nbit) consumes
    nbit/32 + 1 words (Int.cpp:988-1001)."""
    jump_bit = min(range_power // 2 + 1, 128)
    rs = np.random.RandomState(0x600DCAFE)
    lo, hi = 2.0 ** (jump_bit - 1.05), 2.0 ** (jump_bit - 0.95)
    nb, left = jump_bit // 32, jump_bit % 32
    for _ in range(100):
        dist = []
        for _i in range(NB_JUMP):
            words = [int(v) for v in rs.randint(0, 2**32, size=nb + 1, dtype=np.uint64)]
            words[nb] &= (1 << left) - 1
            v = sum(w << (32 * k) for k, w in enumerate(words))
            dist.append(v or 1)
        if lo < sum(dist) / NB_JUMP < hi:
            break
    pts = [ec.mul(d) for d in dist]
    return dist, [p[0] for p in pts], [p[1] for p in pts]


def dp_mask(bits):
    """Kangaroo::SetDP (Kangaroo.cpp:154-164)"""
    return 0 if bits == 0 else (~((1 << (64 - min(bits, 64))) - 1)) & 0xFFFFFFFFFFFFFFFF


class Solver:
    def __init__(self, start, end, pub, dp_bits, grid=None, max_found=1 << 17, seed=None, ingest_threads=0):
        import torch
        self.torch = torch
        self.rank = int(os.environ.get("RANK", "0"))
        self.world = int(os.environ.get("WORLD_SIZE", "1"))
        self.local = int(os.environ.get("LOCAL_RANK", "0"))
        torch.cuda.set_device(self.local)
        self.dist = None
        if self.world > 1:
            import torch.distributed as dist
            if not dist.is_initialized():
                dist.init_process_group("nccl", device_id=torch.device("cuda", self.local))
            self.dist = dist
        self.start, self.end, self.pub, self.dp_bits = start, end, pub, dp_bits
        width = end - start
        self.range_power = width.bit_length()                         # Kangaroo::InitRange (:877-890)
        self.wdiv2 = width >> 1
        # Kangaroo::InitSearchKey (:892-909): keyToSearch = P - start*G
        self.key = ec.add(pub, ec.neg(ec.mul(start))) if start else pub
        gx, gy = grid or GPUEngine.GetGridSize(self.local, 0, 0)
        self.eng = GPUEngine(gx, gy, self.local, max_found)
        self.table = create_jump_table(self.range_power)
        self.eng.SetParams(dp_mask(dp_bits), *self.table)
        self.eng.SetWildOffset(self.wdiv2)
        # Kangaroo::CreateHerd (:670-738): tame d in [0, 2^rangePower), wild d - width/2; points on the device
        n = self.eng.nbKangaroo
        self.rng = np.random.Generator(np.random.PCG64((seed if seed is not None else int(time.time())) * 1000 + self.rank))
        sc, d128 = random_herd_arrays(n, self.range_power, self.wdiv2, self.rng)
        self.eng.CreateHerdRaw(sc, d128, self.key)
        self.gather = DPGather(self.eng, self.dist, self.rank, self.world, torch, wire="dp40") if self.world > 1 else None
        self.dps = DPTable(threads=ingest_threads) if self.rank == 0 else None      # rank 0: the reference HashTable
        # Two pinned staging buffers: while the ingest thread inserts step k's records, step k+1's land in the other one.  The
        # NCCL kernels of a step cannot start before the jump launch that occupies every SM has finished, so without this
        # decoupling the CPU insert would sit exposed between two launches.
        self._hosts = ([torch.empty(self.world * max_found * DP40_BYTES, dtype=torch.uint8).pin_memory() for _ in range(2)]
                       if self.rank == 0 else None)
        self._hidx = 0
        self._work = queue.Queue(maxsize=1)
        self._done = queue.Queue()
        self._pending = 0
        self._acc_found, self._acc_resets = None, []
        self._thread = None
        if self.rank == 0:
            self._thread = threading.Thread(target=self._ingest_loop, daemon=True)
            self._thread.start()
        self._ctrl = torch.zeros(2 + 2 * MAX_RESETS, dtype=torch.int64, device="cuda")
        self.jumps = 0
        self.same_herd = 0
        self.resets_done = 0
        self.t_ingest = 0.0
        self.stop = False

    # -- rank 0: ingest -------------------------------------------------------------------------------------------
    def _ingest(self, segments):
        """segments: list of (rank, uint8 numpy view of that rank's 40-byte records).  Returns (key or None, resets)."""
        found, resets = None, []
        t0 = time.perf_counter()
        for r, buf in segments:
            if buf.size == 0:
                continue
            for kind, rk, kidx, d_old, d_new in self.dps.add_dp40(buf, r):
                if kind == EV_COLLISION and found is None:
                    found = self.dps.resolve(d_old, d_new, self.key, self.start)     # Kangaroo.cpp:255-302
                    if found is None:
                        resets.append((rk, kidx))                                    # "unexpected wrong collision, reset kangaroo"
                elif kind == EV_RESET:
                    resets.append((rk, kidx))
        self.t_ingest += time.perf_counter() - t0
        return found, resets

    def _ingest_loop(self):
        while True:
            segs = self._work.get()
            if segs is None:
                return
            self._done.put(self._ingest(segs))

    def _submit(self, segs):
        """hand one step's records to the ingest thread"""
        self._work.put(segs)
        self._pending += 1

    def _staging(self):
        """the staging buffer for this step; at most one older step may still be in the ingest thread (it reads the OTHER buffer)"""
        while self._pending >= 2:
            self._take(block=True)
        host = self._hosts[self._hidx]
        self._hidx ^= 1
        return host

    def _take(self, block):
        f, r = self._done.get(block=block)
        self._pending -= 1
        if self._acc_found is None:
            self._acc_found = f
        self._acc_resets += r

    def _harvest(self, wait_all=False):
        """results of the inserts finished so far -> (key or None, resets)"""
        while self._pending and (wait_all or not self._done.empty()):
            self._take(block=True)
        found, resets = self._acc_found, self._acc_resets
        self._acc_found, self._acc_resets = None, []
        return found, resets

    def _reset_kangaroo(self, kidx):
        """Kangaroo.cpp:601-609: CreateHerd(1, type) + SetKangaroo(kIdx) on the owning engine."""
        v = int(self.rng.integers(0, 1 << 62)) | (int(self.rng.integers(0, 1 << 62)) << 62) | (int(self.rng.integers(0, 1 << 62)) << 124)
        v &= (1 << self.range_power) - 1
        if kidx % 2 == WILD:
            d = (v - self.wdiv2) % ORDER
            pos = ec.add(self.key, ec.mul(d))
        else:
            d = v
            pos = ec.mul(d)
        if pos is None:
            return
        self.eng.SetKangaroo(kidx, pos[0], pos[1], d)
        self.resets_done += 1

    def step(self):
        """one Launch on every rank; returns the private key on rank 0 when found (None otherwise)"""
        torch = self.torch
        n_found = self.eng.collect_count(relaunch=True)                  # launch i done, launch i+1 running
        cnt = min(n_found, self.eng.maxFound)
        self.jumps += self.eng.nbKangaroo * NB_RUN * self.world
        found, resets = None, []
        if self.gather is not None:
            res = self.gather.step_flat(cnt)                                # rank 0: (counts, cap, device tensor [world*cap*40])
            if self.rank == 0:
                counts, cap, flat = res
                nbytes = self.world * cap * DP40_BYTES
                host = self._staging()
                host[:nbytes].copy_(flat[:nbytes], non_blocking=True)
                torch.cuda.current_stream().synchronize()
                h = host.numpy()
                self._submit([(r, h[r * cap * DP40_BYTES: r * cap * DP40_BYTES + counts[r] * DP40_BYTES]) for r in range(self.world)])
        else:
            if cnt:
                ptr = self.eng.convert_dps_device_ptr()
                dev = torch.as_tensor(SlabView(ptr + 4, cnt * DP40_BYTES), device="cuda")
                host = self._staging()
                host[:cnt * DP40_BYTES].copy_(dev, non_blocking=True)
                torch.cuda.current_stream().synchronize()
                self._submit([(0, host.numpy()[:cnt * DP40_BYTES])])
        if self.rank == 0:
            found, resets = self._harvest()
        # control word: stop flag + kangaroos to re-create, back to their owners
        if self.dist is not None:
            if self.rank == 0:
                resets = resets[:MAX_RESETS]
                c = [1 if found is not None else 0, len(resets)] + [v for rk in resets for v in rk]
                self._ctrl[:len(c)].copy_(torch.tensor(c, dtype=torch.int64))
            self.dist.broadcast(self._ctrl, 0)
            c = self._ctrl.cpu().tolist()
            self.stop = bool(c[0])
            resets = [(c[2 + 2 * i], c[3 + 2 * i]) for i in range(c[1])]
        else:
            self.stop = found is not None
        for rk, kidx in resets:
            self.same_herd += 1
            if rk == self.rank and not self.stop:
                self._reset_kangaroo(kidx)
        return found

    def run(self, max_steps=1 << 30, verbose=True):
        self.eng.callKernel()
        t0 = time.time()
        key = None
        steps = 0
        self.steady = None                      # (time, jumps) after the first 32 steps: NCCL communicator set-up, first table growth
        for s in range(max_steps):
            key = self.step()
            steps += 1
            if steps == 32:
                self.steady = (time.time(), self.jumps)
            if verbose and self.rank == 0 and (s % 64 == 63 or self.stop):
                dt = time.time() - t0
                print("[%6.1fs] 2^%.2f jumps  %.0f MJump/s  %d DPs  dead %d  ingest %.1f ms/step" %
                      (dt, np.log2(max(self.jumps, 1)), self.jumps / dt / 1e6, len(self.dps), self.same_herd,
                       1e3 * self.t_ingest / steps), flush=True)
            if self.stop:
                break
        self.eng.sync()
        if self.rank == 0 and key is None:                      # the last steps' records may still be in the ingest thread
            key, _ = self._harvest(wait_all=True)
        t1 = time.time()
        self.elapsed = t1 - t0
        self.steps = steps
        self.steady_rate = ((self.jumps - self.steady[1]) / (t1 - self.steady[0]) if self.steady and steps > 64 else self.jumps / self.elapsed)
        return key

    def close(self):
        if self._thread is not None:
            self._harvest(wait_all=True)
            self._work.put(None)
            self._thread.join(timeout=10)
            self._thread = None
        self.eng.close()
        if self.dps is not None:
            self.dps.close()


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("config")
    ap.add_argument("--dp", type=int, default=12)
    ap.add_argument("--grid", default="")
    ap.add_argument("--seed", type=int, default=None)
    ap.add_argument("--max-steps", type=int, default=1 << 30)
    ap.add_argument("--ingest-threads", type=int, default=0, help="workers of the rank-0 DP table (0 = min(8, cores))")
    ap.add_argument("--save-work", default="", help="write the rank-0 DP table as a reference work file (HEADW) at the end")
    a = ap.parse_args(argv)
    start, end, pubs = ec.parse_config(a.config)
    grid = tuple(int(v) for v in a.grid.split(",")) if a.grid else None
    rc = 0
    for i, pub in enumerate(pubs):
        s = Solver(start, end, pub, a.dp, grid, seed=a.seed, ingest_threads=a.ingest_threads)
        if s.rank == 0:
            print("Range width: 2^%d  kangaroos/GPU: %d  GPUs: %d  dp: %d  ingest threads: %d" %
                  (s.range_power, s.eng.nbKangaroo, s.world, a.dp, s.dps.threads), flush=True)
        key = s.run(a.max_steps)
        if s.rank == 0:
            print("Solver rate: %.0f MJump/s steady state (after the first 32 steps), %.0f MJump/s over all %d steps (%.2f s); "
                  "rank-0 ingest %.2f ms/step; %d DPs; %d dead kangaroos re-created" %
                  (s.steady_rate / 1e6, s.jumps / s.elapsed / 1e6, s.steps, s.elapsed, 1e3 * s.t_ingest / max(s.steps, 1), len(s.dps), s.same_herd))
            if a.save_work:
                s.dps.save_work(a.save_work, a.dp, start, end, pub, total_count=s.jumps, total_time=s.elapsed)
                print("work file written: %s" % a.save_work)
            if key is not None and ec.mul(key) == pub:
                print("Key#%2d Pub:  0x%064X\n       Priv: 0x%X" % (i, pub[0], key))
            else:
                print("Key#%2d not found" % i); rc = 1
        s.close()
    try:
        import torch.distributed as dist
        if dist.is_initialized():
            dist.destroy_process_group()
    except Exception:
        pass
    return rc


if __name__ == "__main__":
    sys.exit(main())
