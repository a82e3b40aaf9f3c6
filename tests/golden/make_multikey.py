"""Writes a seeded multi-key solver input: a range of 2^BITS, K public keys in it, and the K private keys in input order.

    python tests/golden/make_multikey.py OUT.txt OUT.answers.txt --keys 64 --bits 64 --seed 1

The input is the reference's config format (Kangaroo::ParseConfigFile): range start, range end, then one compressed
public key per line, all hex."""
import argparse
import os
import random
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from kangaroo_b200 import ecmath as ec  # noqa: E402


def make(keys, bits, seed):
    """-> (start, end, [priv ...]) drawn from random.Random(seed)"""
    rng = random.Random(seed)
    start = rng.getrandbits(255) >> bits << bits
    end = start + (1 << bits) - 1
    return start, end, [start + rng.getrandbits(bits) for _ in range(keys)]


def write(cfg, answers, start, end, privs):
    lines = ["%X" % start, "%X" % end]
    for k in privs:
        x, y = ec.mul(k)
        lines.append("%02X%064X" % (2 + (y & 1), x))
    with open(cfg, "w") as f:
        f.write("\n".join(lines) + "\n")
    with open(answers, "w") as f:
        f.write("\n".join("%064X" % k for k in privs) + "\n")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("config")
    ap.add_argument("answers")
    ap.add_argument("--keys", type=int, default=64)
    ap.add_argument("--bits", type=int, default=64)
    ap.add_argument("--seed", type=int, default=1)
    a = ap.parse_args()
    write(a.config, a.answers, *make(a.keys, a.bits, a.seed))
