"""-m gpu: the DP server.  kgx_resolver_verify against an ecmath model of the check, then the server as a process: the table it
writes against an in-process DeviceDPTable, solves through it with the reference's CPU client and the drop-in GPU client, and
its saves, resumes and full table.  Every socket is on 127.0.0.1; every process is killed and waited for at the end.  Tests
that need oracle/_ref/kangaroo_ref_cpu or build/kangaroo_b200 skip without them."""
import os
import re
import struct
import subprocess
import sys
import time

import numpy as np
import pytest

from kangaroo_b200 import ecmath as ec
from tests.server_util import ROOT, Client, ServerProc, corrupt, engine_records

pytestmark = pytest.mark.gpu
REF_CPU = os.path.join(ROOT, "oracle", "_ref", "kangaroo_ref_cpu")
DROPIN = os.path.join(ROOT, "build", "kangaroo_b200")
START = 1 << 40
END = START + (1 << 44) - 1                                   # a 2^44 range
PRIV = START + 0x5A5A1234567
KEY = ec.mul(PRIV)
KOFF = PRIV - START                                           # K = KEY - START*G = KOFF*G
K = ec.mul(KOFF)
M126 = (1 << 126) - 1


def need(path):
    if not os.path.exists(path):
        pytest.skip("%s not built (needs the reference sources at build time)" % os.path.relpath(path, ROOT))


def tag(m, wild=False, neg=False):
    return m | (int(wild) << 126) | (int(neg) << 127)


def point_of(d):
    """the check's S for a tagged distance"""
    S = ec.mul(d & M126)
    if d >> 127:
        S = ec.neg(S)
    if (d >> 126) & 1:
        S = ec.add(S, K)
    return S


def good_model(rec):
    h = struct.unpack_from("<I", rec, 4)[0]
    x = int.from_bytes(rec[8:24], "little")
    S = point_of(int.from_bytes(rec[24:40], "little"))
    return h < (1 << 18) and S is not None and (S[0] >> 128) & 0x3FFFF == h and S[0] & ((1 << 128) - 1) == x


def rec(d, kidx=7, dh=0, dx=0):
    """the record of tagged distance d (h and x of its S, (0, 0) at infinity), h xor dh, x xor dx"""
    S = point_of(d)
    h, x = ((S[0] >> 128) & 0x3FFFF, S[0] & ((1 << 128) - 1)) if S is not None else (0, 0)
    return struct.pack("<II", kidx, h ^ dh) + (x ^ dx).to_bytes(16, "little") + d.to_bytes(16, "little")


def crafted():
    rs = np.random.RandomState(11)
    m = lambda: int(rs.randint(1, 2**62)) << 62 | int(rs.randint(0, 2**62))
    recs = [rec(tag(m())), rec(tag(m(), neg=True)), rec(tag(m(), wild=True)), rec(tag(m(), wild=True, neg=True)),
            rec(tag(m()), dx=1), rec(tag(m(), wild=True), dx=1 << 127), rec(tag(m()), dx=1 << 64), rec(tag(m(), wild=True), dh=1),
            rec(tag(m()), dh=1 << 18), rec(tag(0)), rec(tag(0, wild=True)), rec(tag(KOFF, wild=True, neg=True)),
            rec(tag(M126)), rec(tag(M126, neg=True)), rec(tag(M126, wild=True)), rec(tag(M126 - 5, wild=True, neg=True))]
    want = [True, True, True, True, False, False, False, False, False, False, True, False, True, True, True, True]
    assert [good_model(r) for r in recs] == want               # the model agrees with what each record was made to be
    return recs, want


@pytest.fixture(scope="module")
def resolver():
    from kangaroo_b200.ingest import DeviceResolver, DPTable
    r = DeviceResolver(DPTable.key_table([K]), START)
    yield r
    r.close()


def check(resolver, recs, want, cap=None, stream=None):
    import torch
    raw = np.frombuffer(b"".join(recs), dtype=np.uint8) if isinstance(recs, list) else recs
    t = torch.from_numpy(raw.copy()).cuda() if raw.size else torch.empty(0, dtype=torch.uint8, device="cuda")
    good, n_bad, idx = resolver.verify(t, cap=cap, stream=stream)
    bad_all = [i for i, w in enumerate(want) if not w]
    keep = raw.reshape(-1, 40)[np.array(want, dtype=bool)] if raw.size else raw
    assert n_bad == len(bad_all)
    assert idx == bad_all[:len(bad_all) if cap is None else cap]
    assert good.cpu().numpy().tobytes() == keep.tobytes()


def test_verify_crafted(resolver):
    recs, want = crafted()
    check(resolver, [], [])
    check(resolver, recs[:1], want[:1])
    check(resolver, recs[4:5], want[4:5])
    check(resolver, recs, want)
    check(resolver, recs, want, cap=3)
    check(resolver, recs, want, cap=0)
    big = [recs[i % len(recs)] for i in range(1000)]                # one group of 1024 records, not filled
    check(resolver, big, [want[i % len(recs)] for i in range(1000)], cap=100)


def test_verify_refuses_a_resolver_of_two_keys():
    import torch
    from kangaroo_b200.ingest import DeviceResolver, DPTable
    r = DeviceResolver(DPTable.key_table([K, ec.G]), START)
    try:
        with pytest.raises(RuntimeError, match="exactly one key"):
            r.verify(torch.zeros(40, dtype=torch.uint8, device="cuda"))
    finally:
        r.close()


def test_verify_refuses_unaligned_scratch(resolver):
    import torch
    recs = torch.zeros(40, dtype=torch.uint8, device="cuda")
    out = torch.empty(40, dtype=torch.uint8, device="cuda")
    small = torch.empty(16, dtype=torch.int32, device="cuda")
    nb = resolver.verify_scratch_bytes(1)
    scratch = torch.empty(nb + 256, dtype=torch.uint8, device="cuda")
    with pytest.raises(RuntimeError, match="256-byte aligned"):
        resolver.verify_raw(recs.data_ptr(), 1, out.data_ptr(), small.data_ptr(), small.data_ptr() + 8, 1, scratch.data_ptr() + 4, nb)


@pytest.fixture(scope="module")
def engine_recs():
    return engine_records(START, END, KEY, 8, 1 << 20, max_found=1 << 19)[:40 << 20]


def test_verify_engine_records(resolver, engine_recs):
    import torch
    n = 1 << 20
    recs = engine_recs.copy().reshape(n, 40)
    planted = [0, 1, 5, 1023, 1024, 4097, 500000, n - 2, n - 1]
    recs[planted] = corrupt(engine_recs, planted)
    want = np.ones(n, dtype=bool)
    want[planted] = False
    raw = recs.reshape(-1)
    check(resolver, raw, want.tolist())
    check(resolver, raw, want.tolist(), cap=4)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)                         # the verify queues behind other work on the side stream
    check(resolver, raw, want.tolist(), stream=side)


def write_cfg(path, start=START, end=END, key=KEY):
    path.write_text("%X\n%X\n04%064X%064X\n" % (start, end, key[0], key[1]))
    return path


def last_counts(text):
    m = re.findall(r"\[Dead (\d+)\]\[Wrong (\d+)\]", text)
    return tuple(int(v) for v in m[-1])


def test_table_equals_in_process_table(tmp_path, engine_recs):
    import torch
    from kangaroo_b200.ingest import DeviceDPTable, EV_RESET
    recs = engine_recs[:40 * 30000].reshape(-1, 40)
    wrong = corrupt(engine_recs, np.arange(100, 140))
    msgs = [recs[:10000], np.concatenate([recs[10000:15000], wrong[:20], recs[15000:20000], wrong[20:]]), recs[20000:30000],
            recs[:300]]                                            # the last one: duplicates, which kill kangaroos
    good = np.concatenate([recs[:30000], recs[:300]])
    srv = ServerProc([write_cfg(tmp_path / "c.txt"), "--dp", 8, "--save-work", tmp_path / "s.work", "--dp-table-capacity", 1 << 20],
                     tmp_path)
    try:
        c = Client(srv.port())
        assert c.config() == (3, START, END, KEY, 8)
        for i, m in enumerate(msgs):
            assert c.send(m, ids=(i, 4242, 1)) == 0
        c.close()
        assert srv.terminate() == 1
    finally:
        srv.close()
    text = srv.text()
    assert re.search(r"  table capacity 1048576 entries \(\d+\.\d\d GB\) on cuda:0\n", text), text[:2000]
    assert "40 wrong DPs of 10040 from 127.0.0.1" in text and "processId 4242, threadId 1, gpuId 1" in text
    t = DeviceDPTable(1 << 20)
    try:
        buf = torch.from_numpy(good.reshape(-1).copy()).cuda()
        evs = t.add(buf.data_ptr(), [len(good)], len(good))
        t.save_work(str(tmp_path / "ref.work"), 8, START, END, KEY)
    finally:
        t.close()
    dead = sum(1 for e in evs if e[0] == EV_RESET)
    assert dead >= 300
    assert last_counts(text) == (dead, 40)
    a, b = (tmp_path / "s.work").read_bytes(), (tmp_path / "ref.work").read_bytes()
    assert a[156:] == b[156:]
    from kangaroo_b200.ingest import read_work_header
    h = read_work_header(str(tmp_path / "s.work"))
    assert (h.dp_bits, h.range_start, h.range_end, h.key, h.total_count) == (8, START, END, KEY, 0)


def run_clients(cmds, cwd, timeout):
    procs, logs = [], []
    try:
        for cmd in cmds:
            log = open(os.path.join(str(cwd), "client%d.log" % len(logs)), "w+")
            logs.append(log)
            procs.append(subprocess.Popen(cmd, stdout=log, stderr=subprocess.STDOUT, cwd=str(cwd)))
        deadline = time.monotonic() + timeout
        for p in procs:
            p.wait(timeout=max(1.0, deadline - time.monotonic()))
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
            p.wait()
    out = []
    for log in logs:
        log.seek(0)
        out.append(log.read())
        log.close()
    return [p.returncode for p in procs], out


def test_reference_cpu_client_solves(tmp_path):
    need(REF_CPU)
    srv = ServerProc([write_cfg(tmp_path / "c.txt"), "--dp", 6, "--dp-table-capacity", 1 << 22], tmp_path)
    try:
        port = srv.port()
        t0 = time.monotonic()
        rcs, outs = run_clients([[REF_CPU, "-t", "2", "-c", "127.0.0.1", "-sp", str(port)]], tmp_path, 600)
        rc = srv.wait(60)
        t_end = time.monotonic()
    finally:
        srv.close()
    text = srv.text()
    assert "Priv: 0x%X" % PRIV in text, text[-3000:]
    assert rcs == [0], outs[0][-2000:]
    assert rc == 0
    assert t_end - t0 < 600


def test_gpu_and_cpu_clients_solve_in56(tmp_path):
    need(REF_CPU)
    need(DROPIN)
    srv = ServerProc([os.path.join(ROOT, "tests", "golden", "in56.txt"), "--dp", 12, "--dp-table-capacity", 1 << 22], tmp_path)
    try:
        port = srv.port()
        rcs, outs = run_clients([[DROPIN, "-t", "0", "-gpu", "-g", "16,128", "-c", "127.0.0.1", "-sp", str(port)],
                                 [REF_CPU, "-t", "2", "-c", "127.0.0.1", "-sp", str(port)]], tmp_path, 600)
        rc = srv.wait(60)
    finally:
        srv.close()
    text = srv.text()
    assert "CD612C0F05F3DA03" in text, text[-3000:]
    assert "[Client 2]" in text or text.count("New connection from") >= 2
    assert rc == 0 and rcs == [0, 0], outs


def entries(text):
    return int(re.findall(r"\]\[(\d+) / \d+ entries\]", text)[-1])


def wait_for(srv, pattern, timeout=120, after=0):
    """the first match of pattern in the server's output from offset `after` on, waited for"""
    deadline = time.monotonic() + timeout
    while time.monotonic() < deadline:
        m = re.search(pattern, srv.text()[after:])
        if m:
            return m
        if srv.p.poll() is not None:
            break
        time.sleep(0.1)
    raise AssertionError("%r not printed:\n%s" % (pattern, srv.text()[-3000:]))


def test_save_resume_and_full_table(tmp_path, engine_recs):
    need(REF_CPU)
    cfg = write_cfg(tmp_path / "c.txt")
    work = tmp_path / "s.work"
    recs = engine_recs.reshape(-1, 40)
    tame = recs[(recs[:, 39] & 0x40) == 0][:8000]                 # tame records only: no hit among them, whatever the order
    srv = ServerProc([cfg, "--dp", 8, "--save-work", work, "--save-interval", 1, "--dp-table-capacity", 1 << 22], tmp_path)
    try:
        c = Client(srv.port())
        for i in range(0, len(tame), 1000):
            assert c.send(tame[i:i + 1000]) in (0, 2)               # OK, or BACKUP while a periodic save runs
        c.close()
        sent = len(srv.text())
        wait_for(srv, r"Work file .* written", after=sent)       # a periodic save after every record was queued
        assert srv.terminate() == 1
    finally:
        srv.close()
    text = srv.text()
    assert "Priv:" not in text
    n = entries(text)
    assert n > 0
    chk = subprocess.run([sys.executable, "-m", "kangaroo_b200.worktool", "check", str(work)], capture_output=True, text=True,
                         timeout=300, cwd=ROOT)
    assert "[100.000% OK]" in chk.stdout, chk.stdout + chk.stderr

    small = ServerProc(["--resume", work, "--dp-table-capacity", 10], tmp_path)
    try:
        assert small.wait(180) == 1
    finally:
        small.close()
    assert "refused" in small.text()

    srv = ServerProc([cfg, "--resume", work, "--dp-table-capacity", 1 << 22], tmp_path)
    try:
        port = srv.port()
        assert "Resume %s: %d DPs" % (work, n) in srv.text()
        rcs, outs = run_clients([[REF_CPU, "-t", "2", "-c", "127.0.0.1", "-sp", str(port)]], tmp_path, 600)
        rc = srv.wait(60)
    finally:
        srv.close()
    assert "Priv: 0x%X" % PRIV in srv.text() and rc == 0 and rcs == [0]


def test_full_table_saves_and_exits_1(tmp_path, engine_recs):
    work = tmp_path / "full.work"
    srv = ServerProc([write_cfg(tmp_path / "c.txt"), "--dp", 8, "--save-work", work, "--dp-table-capacity", 1000], tmp_path)
    try:
        c = Client(srv.port())
        c.send(engine_recs[:40 * 600])
        wait_for(srv, r"\]\[600 / 1000 entries\]")              # the first message is in the table before the second is sent
        c.send(engine_recs[40 * 600:40 * 1600])
        rc = srv.wait(120)
    finally:
        srv.close()
    text = srv.text()
    assert rc == 1
    assert "DP table full" in text and "--dp-table-capacity 2000" in text
    assert "(600 entries, capacity 1000; this batch brought 1000 more)" in text
    from kangaroo_b200.ingest import read_work_header
    assert read_work_header(str(work)).key == KEY
    assert "Work file %s written: 600 DPs" % work in text
    assert read_work_header(str(work)).total_count == 0
