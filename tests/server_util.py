"""Helpers of the DP server's tests and of scripts/server_rate.py: the server as a process, a protocol client in Python, and
valid DP records made by the jump engine itself."""
import os
import re
import signal
import socket
import struct
import subprocess
import sys
import tempfile
import time

import numpy as np

from kangaroo_b200 import ecmath as ec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DP_MAGIC = 0x67DEDDC1


def engine_records(start, end, pub, dp, n, grid=(64, 128), max_found=1 << 18, seed=1):
    """at least n 40-byte DP records (uint8 array, kgx_convert_dps's form) of the search (start, end, pub) at dp, made by the
    engine on cuda:0 from a random herd: every one passes the server's check"""
    import torch
    from kangaroo_b200.dist import SlabView
    from kangaroo_b200.engine import GPUEngine, random_herd_arrays
    from kangaroo_b200.solver import create_jump_table, dp_mask
    width = end - start
    rp, wdiv2 = width.bit_length(), width >> 1
    K = ec.add(pub, ec.neg(ec.mul(start))) if start else pub
    eng = GPUEngine(grid[0], grid[1], 0, max_found)
    try:
        eng.SetParams(dp_mask(dp), *create_jump_table(rp))
        eng.SetWildOffset(wdiv2)
        sc, d128 = random_herd_arrays(eng.nbKangaroo, rp, wdiv2, np.random.Generator(np.random.PCG64(seed)))
        eng.CreateHerdRaw(sc, d128, K)
        eng.callKernel()
        parts, total = [], 0
        while total < n:
            eng.collect_count(relaunch=True)
            raw = torch.as_tensor(SlabView(eng.convert_dps_device_ptr(), 4 + max_found * 40), device="cuda").cpu().numpy()
            cnt = min(int(raw[:4].view(np.uint32)[0]), max_found)
            parts.append(raw[4:4 + 40 * cnt].copy())
            total += cnt
        eng.sync()
    finally:
        eng.close()
    return np.concatenate(parts)


def corrupt(recs, idx):
    """copies of records idx with a bit of x flipped (a wrong record of the right shape)"""
    r = recs.reshape(-1, 40)[idx].copy()
    r[:, 8] ^= 1
    return r


class ServerProc:
    """python -m kangaroo_b200.server on 127.0.0.1, port 0, output to a file; always killed and waited for by close()"""

    def __init__(self, args, cwd, env=None):
        self.log = tempfile.TemporaryFile(mode="w+")
        e = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
        e.update(env or {})
        self.p = subprocess.Popen([sys.executable, "-m", "kangaroo_b200.server"] + [str(a) for a in args] +
                                  ["--bind", "127.0.0.1", "--port", "0"], stdout=self.log, stderr=subprocess.STDOUT, cwd=str(cwd),
                                  env=e)

    def text(self):
        self.log.seek(0)
        return self.log.read()

    def port(self, timeout=180):
        deadline = time.monotonic() + timeout
        while time.monotonic() < deadline:
            m = re.search(r"listening to TCP port (\d+)", self.text())
            if m:
                return int(m.group(1))
            if self.p.poll() is not None:
                raise RuntimeError("the server exited %d before listening:\n%s" % (self.p.returncode, self.text()[-3000:]))
            time.sleep(0.1)
        raise RuntimeError("the server did not listen within %d s:\n%s" % (timeout, self.text()[-3000:]))

    def wait(self, timeout):
        return self.p.wait(timeout=timeout)

    def terminate(self, timeout=120):
        self.p.send_signal(signal.SIGTERM)
        return self.p.wait(timeout=timeout)

    def close(self):
        if self.p.poll() is None:
            self.p.kill()
        self.p.wait()


class Client:
    """the protocol's client side, for tests and the rate script"""

    def __init__(self, port, timeout=60):
        self.s = socket.create_connection(("127.0.0.1", port), timeout=timeout)

    def recv(self, n):
        buf = b""
        while len(buf) < n:
            k = self.s.recv(n - len(buf))
            if not k:
                raise EOFError("server closed the connection")
            buf += k
        return buf

    def config(self):
        self.s.sendall(b"\0")
        raw = self.recv(136)
        v = lambda o: int.from_bytes(raw[o:o + 32], "little")
        return struct.unpack_from("<I", raw)[0], v(4), v(36), (v(68), v(100)), struct.unpack_from("<i", raw, 132)[0]

    def send(self, recs, ids=(0, 0, 0)):
        """one SENDDP message -> the status the server answered"""
        recs = np.ascontiguousarray(recs, dtype=np.uint8).reshape(-1)
        self.s.sendall(b"\2" + struct.pack("<5I", DP_MAGIC, recs.size // 40, *ids))
        self.s.sendall(memoryview(recs))
        return struct.unpack("<i", self.recv(4))[0]

    def status(self):
        self.s.sendall(b"\1")
        return struct.unpack("<i", self.recv(4))[0]

    def close(self):
        self.s.close()
