"""The DP server's protocol layer (kangaroo_b200.server.Server) with a fake sink in place of the GPU path: the reference's CPU
client against it, and raw-socket cases of every command.  No GPU needed.  Every socket is on 127.0.0.1; every process runs
under a timeout and is killed and waited for at the end."""
import os
import socket
import struct
import subprocess
import sys
import threading
import time

import numpy as np
import pytest

from kangaroo_b200 import ecmath as ec
from kangaroo_b200 import server as srv

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_CPU = os.path.join(ROOT, "oracle", "_ref", "kangaroo_ref_cpu")
START, END = 0x10000000000, 0x1FFFFFFFFFF               # a 2^40 range
PRIV = 0x1A2B3C4D5E6
KEY = ec.mul(PRIV)


class FakeSink:
    """keeps every message; answers END once it holds end_after records"""

    def __init__(self, end_after=None):
        self.msgs, self.resets = [], 0
        self.end_after = end_after
        self.lock = threading.Lock()

    def records(self):
        with self.lock:
            return b"".join(b for _, b in self.msgs)

    def put(self, msg, chunks):
        with self.lock:
            self.msgs.append((msg, b"".join(c.tobytes() for c in chunks)))

    def status(self):
        n = len(self.records()) // 40
        return srv.STATUS_END if self.end_after is not None and n >= self.end_after else srv.STATUS_OK

    def reset_dead(self):
        self.resets += 1


@pytest.fixture
def served(tmp_path):
    """-> factory(sink) -> (Server listening on 127.0.0.1 port 0, its output lines); closed at teardown"""
    made = []

    def make(sink, **kw):
        lines = []
        s = srv.Server(START, END, KEY, 10, sink, bind="127.0.0.1", port=0, workdir=str(tmp_path), out=lines.append, **kw)
        s.listen()
        made.append(s)
        return s, lines

    yield make
    for s in made:
        s.close()


def connect(port):
    c = socket.create_connection(("127.0.0.1", port), timeout=10)
    return c


def recv_exact(c, n):
    buf = b""
    while len(buf) < n:
        k = c.recv(n - len(buf))
        if not k:
            raise EOFError("closed after %d of %d bytes" % (len(buf), n))
        buf += k
    return buf


def closed(c):
    """the server closed the connection (EOF or reset) within the socket's timeout"""
    try:
        return c.recv(1) == b""
    except ConnectionResetError:
        return True


def get_config(c):
    c.sendall(bytes([srv.CMD_GETCONFIG]))
    raw = recv_exact(c, 4 + 4 * 32 + 4)
    v = lambda o: int.from_bytes(raw[o:o + 32], "little")
    return struct.unpack_from("<I", raw)[0], v(4), v(36), (v(68), v(100)), struct.unpack_from("<i", raw, 132)[0]


def send_dps(c, recs, magic=srv.DP_MAGIC, n=None, ids=(1, 2, 3)):
    n = len(recs) // 40 if n is None else n
    c.sendall(bytes([srv.CMD_SENDDP]) + struct.pack("<5I", magic, n, *ids) + recs)


def check_record(rec, K):
    """the server's rule on one 40-byte record, in Python: S = +-|d|*G (+ K when the type bit is set)"""
    h = struct.unpack_from("<I", rec, 4)[0]
    x = int.from_bytes(rec[8:24], "little")
    d = int.from_bytes(rec[24:40], "little")
    S = ec.mul(d & ((1 << 126) - 1))
    if d >> 127:
        S = ec.neg(S)
    if (d >> 126) & 1:
        S = ec.add(S, K)
    return h < (1 << 18) and S is not None and (S[0] >> 128) & 0x3FFFF == h and S[0] & ((1 << 128) - 1) == x


def test_reference_cpu_client(served, tmp_path):
    if not os.path.exists(REF_CPU):
        pytest.skip("oracle/_ref/kangaroo_ref_cpu not built (needs the reference sources at build time)")
    sink = FakeSink(end_after=64)
    s, lines = served(sink)
    log = open(tmp_path / "client.log", "w+")
    p = subprocess.Popen([REF_CPU, "-t", "2", "-c", "127.0.0.1", "-sp", str(s.port)], stdout=log, stderr=subprocess.STDOUT,
                         cwd=str(tmp_path))
    knb = []
    try:
        deadline = time.monotonic() + 120
        while p.poll() is None and time.monotonic() < deadline:
            with s._lock:
                knb += [c.knb for c in s.clients if c.knb]
            time.sleep(0.05)
        rc = p.poll()
    finally:
        if p.poll() is None:
            p.kill()
        p.wait()
    log.seek(0)
    text = log.read()
    assert rc is not None, "the client did not exit after END:\n" + text[-2000:]
    assert "Succesfully connected to server" in text, text[-2000:]
    assert any("New connection from 127.0.0.1" in ln for ln in lines)
    assert 2 * 1024 in knb                                    # SETKNB: 2 threads x CPU_GRP_SIZE kangaroos
    recs = sink.records()
    assert len(recs) >= 64 * 40 and len(recs) % 40 == 0
    K = ec.add(KEY, ec.neg(ec.mul(START)))
    bad = [i for i in range(min(len(recs) // 40, 96)) if not check_record(recs[40 * i:40 * i + 40], K)]
    assert bad == []


def test_config_and_status(served):
    sink = FakeSink()
    s, _ = served(sink)
    with connect(s.port) as c:
        assert get_config(c) == (3, START, END, KEY, 10)
        c.sendall(bytes([srv.CMD_STATUS]))
        assert struct.unpack("<i", recv_exact(c, 4))[0] == srv.STATUS_OK
        c.sendall(bytes([srv.CMD_SETKNB]) + struct.pack("<Q", 12345))
        c.sendall(bytes([srv.CMD_STATUS]))
        recv_exact(c, 4)
        assert s.kangaroos() == 12345
    deadline = time.monotonic() + 5
    while s.n_clients() and time.monotonic() < deadline:
        time.sleep(0.02)
    assert s.kangaroos() == 0                                 # dropped with its connection


@pytest.mark.parametrize("magic,n", [(0x12345678, 3), (srv.DP_MAGIC, 0)])
def test_bad_dp_header_closes_that_connection_only(served, magic, n):
    sink = FakeSink()
    s, lines = served(sink)
    good = bytes(range(40)) * 2
    with connect(s.port) as a, connect(s.port) as b:
        assert get_config(b)[0] == 3
        send_dps(a, b"", magic=magic, n=n)
        assert closed(a)
        send_dps(b, good)
        assert struct.unpack("<i", recv_exact(b, 4))[0] == srv.STATUS_OK
        assert get_config(b)[0] == 3
    assert sink.records() == good
    assert any("Closing connection" in ln for ln in lines)


def test_message_larger_than_a_chunk(served, monkeypatch):
    monkeypatch.setattr(srv, "CHUNK_RECORDS", 7)
    sink = FakeSink()
    s, _ = served(sink)
    recs = np.random.RandomState(5).randint(0, 256, 20 * 40, dtype=np.uint8).tobytes()
    with connect(s.port) as c:
        send_dps(c, recs, ids=(7, 8, 9))
        assert struct.unpack("<i", recv_exact(c, 4))[0] == srv.STATUS_OK
    assert sink.records() == recs
    msg = sink.msgs[0][0]
    assert (msg.n, msg.thread_id, msg.process_id, msg.gpu_id) == (20, 7, 8, 9)


def test_large_message_with_real_chunks(served):
    sink = FakeSink()
    s, _ = served(sink)
    n = srv.CHUNK_RECORDS + 3
    recs = np.arange(n * 10, dtype=np.uint32).tobytes()
    with connect(s.port) as c:
        c.settimeout(60)
        send_dps(c, recs)
        assert struct.unpack("<i", recv_exact(c, 4))[0] == srv.STATUS_OK
    assert sink.records() == recs


def test_reset_dead(served):
    sink = FakeSink()
    s, _ = served(sink)
    with connect(s.port) as c:
        c.sendall(b"R\0\0")
        assert recv_exact(c, 3) == b"OK\n"
    assert sink.resets == 1


def save_kang(c, name, dists, checksum=None):
    raw = b"".join(int(d).to_bytes(16, "little") for d in dists)
    total = sum(dists) % (1 << 256) if checksum is None else checksum
    c.sendall(bytes([srv.CMD_SAVEKANG]) + struct.pack("<I", len(name)) + name + struct.pack("<Q", len(dists)))
    for o in range(0, len(raw), 16 * srv.KANG_PER_BLOCK):
        c.sendall(raw[o:o + 16 * srv.KANG_PER_BLOCK])
    c.sendall(total.to_bytes(32, "little"))


def load_kang(c, name):
    c.sendall(bytes([srv.CMD_LOADKANG]) + struct.pack("<I", len(name)) + name)
    n = struct.unpack("<Q", recv_exact(c, 8))[0]
    if n == 0:
        return []
    raw = recv_exact(c, 16 * n)
    total = int.from_bytes(recv_exact(c, 32), "little")
    dists = [int.from_bytes(raw[16 * i:16 * i + 16], "little") for i in range(n)]
    assert total == sum(dists) % (1 << 256)
    return dists


def test_kangaroo_files_round_trip(served, tmp_path):
    sink = FakeSink()
    s, lines = served(sink)
    rs = np.random.RandomState(3)
    dists = [int(rs.randint(0, 2**62)) << 64 | int(rs.randint(0, 2**62)) for _ in range(5000)] + [(1 << 128) - 1]
    with connect(s.port) as c:
        save_kang(c, b"kang.wss", dists)
        get_config(c)                                         # the save is complete before the next command is read
        raw = (tmp_path / "kang.wss").read_bytes()
        assert struct.unpack_from("<IIQ", raw) == (srv.HEADKS, 0, len(dists))
        assert len(raw) == 16 + 16 * len(dists)
        assert load_kang(c, b"kang.wss") == dists
        save_kang(c, b"other.wss", dists[:10], checksum=12345)
        get_config(c)
        assert load_kang(c, b"missing.wss") == []
    assert not (tmp_path / "other.wss").exists() and not (tmp_path / "other.wss.tmp").exists()
    assert any("wrong checksum" in ln for ln in lines)


@pytest.mark.parametrize("name", [b"../escape.wss", b"sub/k.wss", b"..", b".", b"a\\b", b"a\0b", b"x" * 256, b""])
def test_kangaroo_file_names_confined(served, tmp_path, name):
    sink = FakeSink()
    work = tmp_path / "work"
    work.mkdir()
    (work / "sub").mkdir()
    s, _ = served(sink)
    s.workdir = str(work)
    before = sorted(p for p in tmp_path.rglob("*"))
    with connect(s.port) as c:
        try:
            save_kang(c, name, [1, 2, 3])
        except OSError:
            pass
        assert closed(c)
    with connect(s.port) as c:
        try:
            c.sendall(bytes([srv.CMD_LOADKANG]) + struct.pack("<I", len(name)) + name)
        except OSError:
            pass
        assert closed(c)
    assert sorted(p for p in tmp_path.rglob("*")) == before


def test_unknown_command_closes(served):
    sink = FakeSink()
    s, lines = served(sink)
    with connect(s.port) as c:
        c.sendall(bytes([9]))
        assert closed(c)
    assert any("unexpected command [9]" in ln for ln in lines)


def test_config_with_two_keys_refused(tmp_path):
    cfg = tmp_path / "two.txt"
    cfg.write_text("%X\n%X\n04%064X%064X\n04%064X%064X\n" % (START, END, KEY[0], KEY[1], ec.G[0], ec.G[1]))
    p = subprocess.run([sys.executable, "-m", "kangaroo_b200.server", str(cfg), "--dp", "10", "--bind", "127.0.0.1", "--port", "0"],
                       capture_output=True, text=True, timeout=120, cwd=ROOT)
    assert p.returncode == 2
    assert "holds 2 keys" in p.stderr and "exactly one key" in p.stderr


def test_dp_required_without_resume(tmp_path):
    cfg = tmp_path / "one.txt"
    cfg.write_text("%X\n%X\n04%064X%064X\n" % (START, END, KEY[0], KEY[1]))
    with pytest.raises(SystemExit):
        srv.parse_args([str(cfg)])
    a, start, end, key, dp = srv.parse_args([str(cfg), "--dp", "14"])
    assert (start, end, key, dp, a.port, a.bind) == (START, END, KEY, 14, srv.DEFAULT_PORT, "0.0.0.0")


def test_file_name_rule():
    assert srv.file_name_error(b"kang.wss") is None
    for bad in (b"", b".", b"..", b"a/b", b"a\\b", b"a\0", b"y" * 256):
        assert srv.file_name_error(bad)


def test_record_queue_budget_blocks_and_batches():
    q = srv.RecordQueue(budget=3 * 40)
    m = object()
    q.put_records(m, [np.zeros(80, np.uint8)])
    done = threading.Event()
    t = threading.Thread(target=lambda: (q.put_records(m, [np.ones(80, np.uint8)]), done.set()))
    t.start()
    assert not done.wait(0.3)                                 # 80 + 80 bytes > the budget of 120: the handler waits
    kind, batch = q.take(1 << 20)
    assert kind == "recs" and len(batch) == 1
    assert done.wait(5)
    t.join()
    q.put_records(m, [np.full(40, 2, np.uint8)])
    q.put("save")
    kind, batch = q.take(2)                                   # 2 + 1 records > 2: the second chunk waits
    assert kind == "recs" and len(batch) == 1 and batch[0][1][0] == 1
    kind, batch = q.take(2)
    assert kind == "recs" and len(batch) == 1 and batch[0][1][0] == 2
    assert q.take(2) == ("save", None)
    assert q.blocked_s > 0.2


def test_server_files_and_links_refused(served, tmp_path):
    """names of the server's own files (work file, its .tmp, config) and symbolic links are refused; nothing changes"""
    sink = FakeSink()
    work = tmp_path / "w"
    work.mkdir()
    (work / "s.work").write_bytes(b"table")
    (work / "c.txt").write_bytes(b"config")
    (tmp_path / "outside").write_bytes(b"secret")
    os.symlink(tmp_path / "outside", work / "link.wss")
    os.symlink(tmp_path / "outside2", work / "dangling.wss.tmp")
    s, lines = served(sink)
    s.workdir = str(work)
    s.protected = srv.Server(0, 1, KEY, 1, sink, protected=[str(work / "s.work"), str(work / "c.txt")]).protected
    for name in (b"s.work", b"s.work.tmp", b"c.txt", b"link.wss", b"dangling.wss"):
        with connect(s.port) as c:
            try:
                save_kang(c, name, [1, 2, 3])
            except OSError:
                pass
            assert closed(c), name
    for name in (b"s.work", b"link.wss"):
        with connect(s.port) as c:
            c.sendall(bytes([srv.CMD_LOADKANG]) + struct.pack("<I", len(name)) + name)
            assert closed(c), name
    assert (work / "s.work").read_bytes() == b"table" and (work / "c.txt").read_bytes() == b"config"
    assert (tmp_path / "outside").read_bytes() == b"secret" and not (tmp_path / "outside2").exists()
    assert sorted(os.listdir(work)) == ["c.txt", "dangling.wss.tmp", "link.wss", "s.work"]
    assert any("symbolic link" in ln for ln in lines) and any("server's own files" in ln for ln in lines)


def test_handler_threads_pruned_and_joined(served):
    sink = FakeSink()
    s, _ = served(sink)
    for _ in range(20):
        with connect(s.port) as c:
            get_config(c)
    deadline = time.monotonic() + 5
    while s.n_clients() and time.monotonic() < deadline:
        time.sleep(0.02)
    with connect(s.port) as c:
        get_config(c)
        assert len(s._handlers) <= 2                          # finished handlers are dropped at the next accept
        s.close()
        assert all(not t.is_alive() for t in s._handlers) and not s._acceptor.is_alive()
