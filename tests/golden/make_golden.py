"""Generate tests/golden/jump_golden.json from the REFERENCE's own code (oracle/_ref/libkref.so, i.e. the
unmodified reference SECPK1 sources driven by oracle/ref_harness.cpp).  Run where oracle/_ref/libkref.so is built:

    python tests/golden/make_golden.py

The fixture is committed, so the tests need neither the reference sources nor oracle/_ref."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import kgo  # noqa: E402


def hx(v):
    return "%X" % v


def main():
    ref = kgo.Reference()
    out = {"generator": "tests/golden/make_golden.py via oracle/_ref/libkref.so (reference @ 37576c8)", "cases": []}
    # Check.cpp:472-483 range; key as VC_CUDA8/in64.txt known answer
    cases = [
        dict(name="check64_dp8", range_power=64, seed=42, n=256, njumps=64, dp=8, first_type=0,
             key_priv=0x5B3F38AF935A3640D158E871CE6E9666DB862636383386EE510F18CCC3BD72EB),
        dict(name="in80_dp4", range_power=80, seed=7, n=128, njumps=128, dp=4, first_type=0,
             key_priv=0xB60E83280258A40F9CDF1649744D730D6E939DE92A2BE19B0F1234567890ABCD),
        dict(name="puzzle110_dp6", range_power=109, seed=110, n=96, njumps=64, dp=6, first_type=1,
             key_priv=0x35C0D7234DF7DEB0F20CF7062444),
    ]
    for c in cases:
        table = ref.create_jump_table(c["range_power"])
        key = ref.ec_mul_g(c["key_priv"])
        wdiv2 = (2 ** c["range_power"] - 1) >> 1
        ref.rseed(c["seed"])
        px, py, d = ref.create_herd(c["n"], c["range_power"], wdiv2, key, c["first_type"])
        start = [(hx(kgo.from_limbs(px[i])), hx(kgo.from_limbs(py[i])), hx(kgo.from_limbs(d[i]))) for i in range(c["n"])]
        mask = (~((1 << (64 - c["dp"])) - 1)) & 0xFFFFFFFFFFFFFFFF
        dps = ref.jump_cpu(px, py, d, table, c["njumps"], mask)
        end = [(hx(kgo.from_limbs(px[i])), hx(kgo.from_limbs(py[i])), hx(kgo.from_limbs(d[i]))) for i in range(c["n"])]
        out["cases"].append(dict(
            name=c["name"], range_power=c["range_power"], seed=c["seed"], n=c["n"], njumps=c["njumps"], dp_bits=c["dp"],
            dp_mask=hx(mask), first_type=c["first_type"], key=[hx(key[0]), hx(key[1])], width_div2=hx(wdiv2),
            jump_table=[[hx(kgo.from_limbs(table[0][i])), hx(kgo.from_limbs(table[1][i])), hx(kgo.from_limbs(table[2][i]))]
                        for i in range(32)],
            start=start, end=end,
            dps=sorted([hx(x), hx(dd), k, j] for (x, dd, k, j) in dps)))
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "jump_golden.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=0)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
