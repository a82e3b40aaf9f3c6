"""Regenerate tests/golden/ref_golden.json: the transcripts of tests/ref_transcripts.py computed by the reference's own
SECPK1 code (oracle/_ref/libkref.so, built by `make -C oracle ref REF=<reference source tree>`).

    python tests/golden/make_ref_golden.py"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import kgo  # noqa: E402
from tests import ref_transcripts as rt  # noqa: E402


def main():
    if not os.path.exists(kgo.Reference.path):
        raise SystemExit("%s is missing: build it with `make -C oracle ref REF=<reference source tree>`" % kgo.Reference.path)
    ref = kgo.Reference()
    runs = {
        "field_ops": rt.field_ops(ref),
        "order_ops": rt.order_ops(ref),
        "rng_and_rand": rt.rng_and_rand(ref),
        "scalar_mult_and_add": rt.scalar_mult_and_add(ref),
        "jump_tables": rt.jump_tables(ref),
        "herd_and_jump_loop": rt.herd_and_jump_loop(ref, grp=1024),
        "hash_convert": rt.hash_convert(ref),
        "symmetric_herd_and_walk": rt.symmetric_herd_and_walk(ref, grp=24)[0],
    }
    for rp in rt.SYM_RANGE_POWERS:
        runs["symmetric_jump_table_%d" % rp] = rt.symmetric_jump_table(ref, rp)
    out = {name: {"sha256": rt.digest(t), "entries": len(t), "head": rt.head(t)} for name, t in runs.items()}
    path = os.path.join(ROOT, "tests", "golden", "ref_golden.json")
    with open(path, "w") as f:
        json.dump({"source": "reference SECPK1 (Int, IntMod, IntGroup, Point, SECP256K1, Random) + HashTable::Convert",
                   "transcripts": out}, f, indent=1)
    print("wrote", path)


if __name__ == "__main__":
    main()
