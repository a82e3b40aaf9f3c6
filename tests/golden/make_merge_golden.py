"""Regenerate the work-file check / merge fixtures with the reference's own CPU program (oracle/_ref/kangaroo_ref_cpu, built
by `make -C oracle ref REF=<reference source tree>`), on ref_work48's key and range (make_work_golden.py):

    ref_work48b.work.gz         a second reference run (its own random herd, dp 16), which together with ref_work48 does
                                not find the key
    ref_merge48.work.gz         the reference's `-wm ref_work48 ref_work48b` output (it ends right after the table)
    ref_work48_bad.work.gz      ref_work48 with corrupted entries (CORRUPTIONS), and in merge_golden.json the wrong count the
                                reference's -wcheck gives for it
    merge_golden.json           that count

The crafted pair whose merge finds the key is built by the tests themselves (tests/test_worktool_cpu.py: crafted_pair).

    python tests/golden/make_merge_golden.py"""
import gzip
import json
import os
import re
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests.golden import make_work_golden as g  # noqa: E402

REFBIN = g.REFBIN
GOLD = os.path.join(ROOT, "tests", "golden")
HEADER = 156
# (bucket rank among the non-empty buckets, entry, what): each corruption hits its own bucket
CORRUPTIONS = [(0, 0, "x_lo_bit"), (1, 0, "x_hi_bit"), (2, 0, "move_bucket"), (3, 0, "type_bit"), (4, 0, "sign_bit_tame"),
               (5, 0, "sign_bit_wild")]


def buckets(raw):
    """[(h, offset of the bucket's first entry, nbItem)] of a HEADW file's table"""
    out, off = [], HEADER
    for h in range(1 << 18):
        nb = int.from_bytes(raw[off:off + 4], "little")
        out.append((h, off + 8, nb))
        off += 8 + 32 * nb
    return out, off


def corrupt(raw):
    """ref_work48 with CORRUPTIONS applied -> bytes (the table keeps its shape: an entry moved to another bucket swaps places
    with that bucket's first entry)"""
    b = bytearray(raw)
    table, _ = buckets(raw)
    full = [t for t in table if t[2] > 0]
    tame = [t for t in full if not (int.from_bytes(raw[t[1] + 24:t[1] + 32], "little") >> 62) & 1]
    wild = [t for t in full if (int.from_bytes(raw[t[1] + 24:t[1] + 32], "little") >> 62) & 1]
    used = set()

    def pick(pool):
        for t in pool:
            if t[0] not in used:
                used.add(t[0])
                return t
        raise SystemExit("not enough non-empty buckets")

    for _, _, what in CORRUPTIONS:
        if what == "x_lo_bit":
            t = pick(full); b[t[1] + 0] ^= 0x10
        elif what == "x_hi_bit":
            t = pick(full); b[t[1] + 15] ^= 0x20
        elif what == "move_bucket":
            t, u = pick(full), pick(full)                    # swap the first entries of two buckets: both are wrong
            b[t[1]:t[1] + 32], b[u[1]:u[1] + 32] = raw[u[1]:u[1] + 32], raw[t[1]:t[1] + 32]
        elif what == "type_bit":
            t = pick(full); b[t[1] + 31] ^= 0x40
        elif what == "sign_bit_tame":
            t = pick(tame); b[t[1] + 31] ^= 0x80               # x(-P) = x(P): stays OK
        elif what == "sign_bit_wild":
            t = pick(wild); b[t[1] + 31] ^= 0x80
    return bytes(b)


def ref_wcheck(path):
    out = subprocess.run([REFBIN, "-t", "4", "-wcheck", path], capture_output=True, text=True, timeout=600).stdout
    m = re.search(r"DP Wrong: (\d+)", out)
    return int(m.group(1)) if m else 0, out


def main():
    if not os.path.exists(REFBIN):
        raise SystemExit("%s is missing: build it with `make -C oracle ref REF=<reference source tree>`" % REFBIN)
    with tempfile.TemporaryDirectory() as tmp:
        a = os.path.join(tmp, "a.work")
        with gzip.open(os.path.join(GOLD, "ref_work48.work.gz"), "rb") as src, open(a, "wb") as dst:
            shutil.copyfileobj(src, dst)
        cfg, b = os.path.join(tmp, "in48.txt"), os.path.join(tmp, "b.work")
        open(cfg, "w").write(g.config_text())
        out = subprocess.run([REFBIN, "-t", "1", "-d", str(g.DP_BITS), "-w", b, "-ws", "-wi", "2", "-m", "0.3", cfg],
                             capture_output=True, text=True, timeout=600).stdout
        if "Priv:" in out or not os.path.exists(b):
            raise SystemExit("the second run found the key or saved nothing; run again:\n" + out)
        m = os.path.join(tmp, "m.work")
        out = subprocess.run([REFBIN, "-wm", a, b, m], capture_output=True, text=True, timeout=600).stdout
        if "Priv:" in out or not os.path.exists(m):
            raise SystemExit("the merge found the key or wrote nothing; run again:\n" + out)
        bad = os.path.join(tmp, "bad.work")
        open(bad, "wb").write(corrupt(open(a, "rb").read()))
        wrong, out = ref_wcheck(bad)
        for src, name in ((b, "ref_work48b.work.gz"), (m, "ref_merge48.work.gz"), (bad, "ref_work48_bad.work.gz")):
            with open(src, "rb") as s, gzip.open(os.path.join(GOLD, name), "wb", compresslevel=9) as d:
                shutil.copyfileobj(s, d)
    json.dump({"ref_work48_bad_wrong": wrong, "corruptions": [c[2] for c in CORRUPTIONS]},
              open(os.path.join(GOLD, "merge_golden.json"), "w"), indent=1)
    print("wrote the fixtures; -wcheck of the corrupted file: %d wrong" % wrong)


if __name__ == "__main__":
    main()
