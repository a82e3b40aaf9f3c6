"""Regenerate tests/golden/ref_work48.work.gz: a work file with kangaroos written by the reference's own CPU program
(oracle/_ref/kangaroo_ref_cpu, built by `make -C oracle ref REF=<reference source tree>`).  One CPU thread = 1,024
kangaroos on a 2^48 window (key below), dp 16, saved every 2 s with -ws and stopped by -m before the key is found.  The
table's 2^18 bucket headers make the file 2 MB of mostly zeros, hence the gzip.

    python tests/golden/make_work_golden.py"""
import gzip
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from kangaroo_b200 import ecmath as ec  # noqa: E402

REFBIN = os.path.join(ROOT, "oracle", "_ref", "kangaroo_ref_cpu")
START = 0x62CE27C8FED90758A834C2CB6E3F19BC8A0B5E7D92C0FC0F5700000000000000
PRIV = START + 0x9A3C5E1F0B7A
RANGE_BITS, DP_BITS = 48, 16
OUT = os.path.join(ROOT, "tests", "golden", "ref_work48.work.gz")


def config_text():
    x, y = ec.mul(PRIV)
    return "%X\n%X\n%s%064X\n" % (START, START + (1 << RANGE_BITS) - 1, "03" if y & 1 else "02", x)


def main():
    if not os.path.exists(REFBIN):
        raise SystemExit("%s is missing: build it with `make -C oracle ref REF=<reference source tree>`" % REFBIN)
    with tempfile.TemporaryDirectory() as tmp:
        cfg, work = os.path.join(tmp, "in48.txt"), os.path.join(tmp, "w48.work")
        open(cfg, "w").write(config_text())
        out = subprocess.run([REFBIN, "-t", "1", "-d", str(DP_BITS), "-w", work, "-ws", "-wi", "2", "-m", "0.3", cfg],
                             capture_output=True, text=True, timeout=600).stdout
        if "Priv:" in out or not os.path.exists(work):
            raise SystemExit("the run found the key or saved nothing; run again:\n" + out)
        with open(work, "rb") as src, gzip.open(OUT, "wb", compresslevel=9) as dst:
            shutil.copyfileobj(src, dst)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
