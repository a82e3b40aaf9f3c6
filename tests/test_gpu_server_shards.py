"""-m gpu: the DP server with its table in shards (--devices).  kgx_resolver_verify_partition against kgx_resolver_verify followed
by kgx_dp_partition, byte for byte; then the server with three shards on one GPU against the one-GPU server fed the same
records: counts, wrong lines, dead count and work files, a key found on a shard past the first, resumes across both modes, a
full shard and a resume too large for a shard; --devices 0,1 where two GPUs are visible, and a real client against two shards
where build/kangaroo_b200 was built.  Every socket is on 127.0.0.1; every process is killed and waited for at the end."""
import ctypes
import os
import re
import struct
import subprocess
import sys
import threading

import numpy as np
import pytest

from kangaroo_b200 import ecmath as ec
from tests.server_util import ROOT, Client, ServerProc, corrupt, engine_records
from tests.test_gpu_server import DROPIN, END, KEY, KOFF, START, entries, last_counts, need, rec, run_clients, tag, wait_for, write_cfg

pytestmark = pytest.mark.gpu
NB = 1 << 18
TILE = 256                                                     # kgx_partition.cuh's tile


# ---- the kernel ------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def resolver():
    from kangaroo_b200.ingest import DeviceResolver, DPTable
    r = DeviceResolver(DPTable.key_table([ec.mul(KOFF)]), START)
    yield r
    r.close()


@pytest.fixture(scope="module")
def engine_recs():
    return engine_records(START, END, KEY, 8, 1 << 20, max_found=1 << 19)[:40 << 20].reshape(-1, 40)


def fused(resolver, src, n, world, stride, cap):
    """kgx_resolver_verify_partition -> (out bytes, counts, bad count, bad indices)"""
    import torch
    rows = world * stride if stride else max(n, 1)
    out = torch.full((rows * 40,), 0xEE, dtype=torch.uint8, device="cuda")
    counts = torch.full((world + 1,), -1, dtype=torch.int32, device="cuda")
    bad = torch.full((max(cap, 1),), -1, dtype=torch.int32, device="cuda")
    nb = resolver.verify_partition_scratch_bytes(n, world)
    scratch = torch.empty(nb, dtype=torch.uint8, device="cuda")
    resolver.verify_partition_raw(src.data_ptr(), n, world, stride, out.data_ptr(), counts.data_ptr(), bad.data_ptr(), cap,
                                  scratch.data_ptr(), nb, torch.cuda.current_stream().cuda_stream)
    c = counts.cpu().tolist()
    return out.cpu().numpy().tobytes(), c[:world], c[world], bad[:min(c[world], cap)].cpu().tolist()


def two_calls(resolver, src, n, world, stride, cap):
    """kgx_resolver_verify, then kgx_dp_partition of its good records -> what fused() returns"""
    import torch
    from kangaroo_b200 import load_library
    lib = load_library()
    good = torch.empty(max(n, 1) * 40, dtype=torch.uint8, device="cuda")
    vc = torch.empty(2, dtype=torch.int32, device="cuda")
    bad = torch.full((max(cap, 1),), -1, dtype=torch.int32, device="cuda")
    nb = resolver.verify_scratch_bytes(n)
    scratch = torch.empty(nb, dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    resolver.verify_raw(src.data_ptr(), n, good.data_ptr(), vc.data_ptr(), bad.data_ptr(), cap, scratch.data_ptr(), nb, st)
    n_good, n_bad = vc.cpu().tolist()
    rows = world * stride if stride else max(n, 1)
    out = torch.full((rows * 40,), 0xEE, dtype=torch.uint8, device="cuda")
    counts = torch.full((world + 1,), -1, dtype=torch.int32, device="cuda")
    ps = torch.empty(int(lib.kgx_dp_partition_scratch_bytes(n_good, world)), dtype=torch.uint8, device="cuda")
    assert lib.kgx_dp_partition(ctypes.c_void_p(good.data_ptr()), n_good, world, stride, ctypes.c_void_p(out.data_ptr()),
                                ctypes.c_void_p(counts.data_ptr()), ctypes.c_void_p(ps.data_ptr()), ps.numel(), ctypes.c_void_p(st)) == 0
    c = counts.cpu().tolist()
    assert c[world] == 0                                       # verify keeps no malformed record
    return out.cpu().numpy().tobytes(), c[:world], n_bad, bad[:min(n_bad, cap)].cpu().tolist()


def compare(resolver, recs, worlds, caps=(None, 3), strides=(0, "n")):
    import torch
    recs = np.ascontiguousarray(recs, dtype=np.uint8).reshape(-1, 40)
    n = len(recs)
    src = torch.from_numpy(recs.reshape(-1).copy()).cuda() if n else torch.empty(40, dtype=torch.uint8, device="cuda")
    for world in worlds:
        for stride in strides:
            stride = n + 5 if stride == "n" else stride
            for cap in caps:
                cap = n if cap is None else cap
                got, want = fused(resolver, src, n, world, stride, cap), two_calls(resolver, src, n, world, stride, cap)
                assert got[1:] == want[1:], (world, stride, cap)
                assert got[0] == want[0], (world, stride, cap)


def with_h(recs, h):
    """copies of the records with h replaced (wrong records of the right shape, unless h is their own)"""
    r = np.array(recs, dtype=np.uint8).reshape(-1, 40)
    r[:, 4:8] = np.asarray(h, dtype=np.uint32).reshape(-1, 1).view(np.uint8)
    return r


def h_of(recs):
    return recs[:, 4:8].copy().view(np.uint32).reshape(-1)


WORLDS = (1, 2, 3, 7, 8, 256)


def test_verify_partition_small(resolver, engine_recs):
    recs = engine_recs[:4 * TILE + 8].copy()
    planted = [0, TILE - 1, TILE, 2 * TILE - 1, 3 * TILE + 5, len(recs) - 1]      # first and last of a tile
    recs[planted] = corrupt(recs, planted)
    recs[[7, 2 * TILE + 1]] = with_h(recs[[7, 2 * TILE + 1]], [NB, 0xFFFFFFFF])     # h >= 2^18
    for n in (0, 1, TILE - 1, TILE, TILE + 1):
        compare(resolver, recs[:n], WORLDS)
    compare(resolver, recs, WORLDS, caps=(None, 3, 0))
    compare(resolver, corrupt(recs, np.arange(TILE + 1)), WORLDS)                    # all bad
    compare(resolver, engine_recs[:TILE + 1], WORLDS)                                # all good


def test_verify_partition_one_owner(resolver, engine_recs):
    h = h_of(engine_recs)
    low, high = engine_recs[h < NB // 8][:700], engine_recs[h >= NB - NB // 8][:700]   # owner 0 / owner 7 of 8, only
    assert len(low) == len(high) == 700
    mixed = np.concatenate([low, corrupt(low, [0, 5])])
    for recs in (low, high, mixed):
        compare(resolver, recs, (2, 7, 8, 256))


def test_verify_partition_2_20(resolver, engine_recs):
    n = 1 << 20
    recs = engine_recs[:n].copy()
    rng = np.random.RandomState(5)
    wrong = np.unique(np.concatenate([rng.choice(n, n // 20, replace=False), [0, 1023, 1024, n - 1]]))
    recs[wrong] = corrupt(recs, wrong)
    recs[wrong[::7]] = with_h(recs[wrong[::7]], NB + wrong[::7])
    compare(resolver, recs, (1, 3, 8), caps=(None, 100))
    compare(resolver, recs, (256,), caps=(None,), strides=(0,))


def test_verify_partition_refusals(resolver):
    import torch
    recs = torch.zeros(80, dtype=torch.uint8, device="cuda")
    buf = torch.empty(4096, dtype=torch.uint8, device="cuda")
    nb = resolver.verify_partition_scratch_bytes(2, 3)
    p = buf.data_ptr()
    for world, stride, scratch, why in ((0, 0, nb, "world"), (257, 0, nb, "world"), (3, 1, nb, "stride"), (3, 0, nb - 1, "scratch")):
        with pytest.raises(RuntimeError, match=why):
            resolver.verify_partition_raw(recs.data_ptr(), 2, world, stride, p, p + 1024, p + 2048, 2, p + 2560, scratch)
    assert resolver.verify_partition_scratch_bytes(1, 0) == 0 and resolver.verify_partition_scratch_bytes(1, 257) == 0


# ---- the server --------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tame(engine_recs):
    """tame engine records of distinct points only: no hit and no dead kangaroo among them whatever the order, so every count
    is the same in any arrival order"""
    t = engine_recs[(engine_recs[:, 39] & 0x40) == 0]
    _, first = np.unique(np.ascontiguousarray(t[:, 4:24]).view("V20").reshape(-1), return_index=True)
    return t[np.sort(first)][:60000]


def messages(tame):
    """tame records in 12 messages, 5 % of the records wrong, then a resend of the first 300 -> (messages, records of the
    resend that were wrong in the first message: they are new then, the rest kill a kangaroo each)"""
    rng = np.random.RandomState(3)
    out, fresh = [], 0
    for i in range(12):
        m = tame[5000 * i:5000 * (i + 1)].copy()
        wrong = rng.choice(len(m), 250, replace=False)
        m[wrong] = corrupt(m, wrong)
        out.append(m)
        if i == 0:
            fresh = int((wrong < 300).sum())
    return out + [tame[:300]], fresh


def wrong_lines(text):
    """the per-message wrong lines, without the client's address"""
    return sorted(re.sub(r"from \S+ ", "from C ", s) for s in re.findall(r"\d+ wrong DPs of .*", text))


def serve(tmp_path, name, args, msgs, senders=1):
    """a server fed msgs (one sender, in order; or `senders` connections sending them round robin at once), stopped by SIGTERM
    once everything is sent -> (return code, output)"""
    srv = ServerProc(args, tmp_path)
    try:
        port = srv.port()
        groups = [msgs[k::senders] for k in range(senders)]

        def send(group, ids):
            c = Client(port)
            for m in group:
                c.send(m, ids=ids)
            c.close()

        threads = [threading.Thread(target=send, args=(g, (k, 77, 0))) for k, g in enumerate(groups)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        rc = srv.terminate()
    finally:
        srv.close()
    text = srv.text()
    (tmp_path / (name + ".log")).write_text(text)
    return rc, text


def outcome(text):
    return entries(text), last_counts(text), wrong_lines(text)


def same_file(a, b):
    """two work files equal byte for byte except the run time in the header (bytes 148..155)"""
    a, b = a.read_bytes(), b.read_bytes()
    assert len(a) == len(b)
    assert a[:148] == b[:148] and a[156:] == b[156:]


def worktool_check(path):
    chk = subprocess.run([sys.executable, "-m", "kangaroo_b200.worktool", "check", str(path)], capture_output=True, text=True,
                         timeout=300, cwd=ROOT)
    assert "[100.000% OK]" in chk.stdout, chk.stdout + chk.stderr


def compare_servers(tmp_path, tame, devices, senders=1):
    cfg = write_cfg(tmp_path / "c.txt")
    msgs, fresh = messages(tame)
    base = [cfg, "--dp", 8, "--dp-table-capacity", 1 << 20]
    rc1, one = serve(tmp_path, "one", base + ["--save-work", tmp_path / "one.work"], msgs, senders)
    rcw, sh = serve(tmp_path, "shards", base + ["--save-work", tmp_path / "shards.work", "--devices", devices], msgs, senders)
    assert rc1 == rcw == 1                                     # stopped by the signal, files written
    assert "Priv:" not in one + sh
    assert "fullest shard" in sh and "shards on cuda:%s" % devices in sh
    o1, ow = outcome(one), outcome(sh)
    assert o1 == ow
    n, (dead, wrong), lines = o1
    assert n == 60000 - 12 * 250 + fresh and dead == 300 - fresh and wrong == 12 * 250 and len(lines) == 12
    assert 0 < fresh < 300
    return tmp_path / "one.work", tmp_path / "shards.work"


def test_three_shards_on_one_gpu_equal_the_one_gpu_server(tmp_path, tame):
    one, sh = compare_servers(tmp_path, tame, "0,0,0")
    same_file(one, sh)
    worktool_check(sh)


def test_four_senders(tmp_path, tame):
    compare_servers(tmp_path, tame, "0,0,0", senders=4)


def test_two_gpus(tmp_path, tame):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU visible")
    one, sh = compare_servers(tmp_path, tame, "0,1")
    same_file(one, sh)


def test_key_found_on_a_later_shard(tmp_path):
    """a tame and a wild record at the same point, in a bucket of shard 2 of 3: the server prints the key as the one-GPU server"""
    rng = np.random.RandomState(9)
    while True:
        m = int(rng.randint(1, 2**62)) << 40 | int(rng.randint(0, 2**40))
        w = rec(tag(m, wild=True), kidx=1)
        if struct.unpack_from("<I", w, 4)[0] >= 2 * NB // 3:
            break
    t = rec(tag(m + KOFF), kidx=2)
    assert t[4:24] == w[4:24]
    msg = np.frombuffer(w + t, dtype=np.uint8)
    cfg = write_cfg(tmp_path / "c.txt")
    texts = []
    for extra in ([], ["--devices", "0,0,0"]):
        srv = ServerProc([cfg, "--dp", 8, "--dp-table-capacity", 1 << 16] + extra, tmp_path)
        try:
            c = Client(srv.port())
            c.send(msg)
            c.close()
            rc = srv.wait(120)
        finally:
            srv.close()
        assert rc == 0
        texts.append(srv.text())
    keys = [re.findall(r"(?m)^.*Priv: 0x[0-9A-F]+.*$", s) for s in texts]
    assert keys[0] and keys[0] == keys[1]
    assert "Priv: 0x%X" % (START + KOFF) in texts[1]


def test_resume_across_modes(tmp_path, tame):
    cfg = write_cfg(tmp_path / "c.txt")
    msgs = messages(tame)[0]
    first, second = msgs[:6], msgs[6:]
    cap = ["--dp-table-capacity", 1 << 20]
    w = lambda name: tmp_path / name
    shards = ["--devices", "0,0,0"]
    assert serve(tmp_path, "a1", [cfg, "--dp", 8, "--save-work", w("a1.work")] + cap, first)[0] == 1
    assert serve(tmp_path, "a3", [cfg, "--dp", 8, "--save-work", w("a3.work")] + cap + shards, first)[0] == 1
    same_file(w("a1.work"), w("a3.work"))
    rc3, t3 = serve(tmp_path, "b3", ["--resume", w("a1.work"), "--save-work", w("b3.work")] + cap + shards, second)
    rc1, t1 = serve(tmp_path, "b1", ["--resume", w("a3.work"), "--save-work", w("b1.work")] + cap, second)
    assert rc1 == rc3 == 1
    assert "Resume %s: %d DPs" % (w("a1.work"), 6 * 4750) in t3 and "Resume %s: %d DPs" % (w("a3.work"), 6 * 4750) in t1
    assert outcome(t1) == outcome(t3)
    same_file(w("b1.work"), w("b3.work"))


def test_full_shard_then_resume(tmp_path, tame):
    cfg = write_cfg(tmp_path / "c.txt")
    work = tmp_path / "full.work"
    srv = ServerProc([cfg, "--dp", 8, "--save-work", work, "--dp-table-capacity", 1000, "--devices", "0,0,0"], tmp_path)
    try:
        c = Client(srv.port())
        c.send(tame[:600])
        wait_for(srv, r"\]\[600 / 3000 entries\]")            # the first message is in the table before the second is sent
        c.send(tame[600:3600])                                  # about 1000 more per shard: one of them overflows
        rc = srv.wait(120)
    finally:
        srv.close()
    text = srv.text()
    assert rc == 1
    m = re.search(r"DP table full, server stopped: shard (\d) of 3 \(buckets \[(\d+), (\d+)\) on cuda:0\) holds (\d+) entries, "
                  r"capacity 1000", text)
    assert m, text[-3000:]
    s, lo, hi = int(m.group(1)), int(m.group(2)), int(m.group(3))
    assert (lo, hi) == (s * NB // 3, (s + 1) * NB // 3)
    assert "--dp-table-capacity 2000" in text
    assert "Work file %s written: 600 DPs" % work in text      # a cut between whole batches: nothing of the second message
    worktool_check(work)

    rc, t = serve(tmp_path, "resumed", ["--resume", work, "--dp-table-capacity", 1 << 16, "--devices", "0,0,0",
                                        "--save-work", tmp_path / "more.work"], [tame[600:3600]])
    assert rc == 1 and "Resume %s: 600 DPs" % work in t
    assert entries(t) == 3600 and last_counts(t) == (0, 0)

    small = ServerProc(["--resume", tmp_path / "more.work", "--dp-table-capacity", 1000, "--devices", "0,0,0"], tmp_path)
    try:
        assert small.wait(180) == 1
    finally:
        small.close()
    text = small.text()
    assert "refused" in text and re.search(r"shard \d of 3, buckets \[\d+, \d+\) on cuda:0", text), text[-2000:]
    assert "listening" not in text


def test_dropin_client_solves_against_two_shards(tmp_path):
    need(DROPIN)
    start, end, pubs = ec.parse_config(os.path.join(ROOT, "tests", "golden", "in40_5.txt"))
    cfg = write_cfg(tmp_path / "c.txt", start, end, pubs[0])
    srv = ServerProc([cfg, "--dp", 12, "--dp-table-capacity", 1 << 22, "--devices", "0,0"], tmp_path)
    try:
        port = srv.port()
        rcs, outs = run_clients([[DROPIN, "-t", "0", "-gpu", "-g", "16,128", "-c", "127.0.0.1", "-sp", str(port)]], tmp_path, 600)
        rc = srv.wait(60)
    finally:
        srv.close()
    text = srv.text()
    m = re.search(r"Priv: 0x([0-9A-F]+)", text)
    assert m, text[-3000:]
    priv = int(m.group(1), 16)
    assert start <= priv <= end and ec.mul(priv) == pubs[0]
    assert rc == 0 and rcs == [0], outs
