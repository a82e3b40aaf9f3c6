#!/bin/bash
# build_ingest.sh -- build/libkgx_ingest.so: the rank-0 DP ingest (kgx_ingest.cpp, C ABI include/kgx_ingest.h) linked
# with the reference's UNMODIFIED HashTable.cpp + SECPK1 + Timer.cpp, compiled where they lie under $REF.
# Needs the reference sources ($REF, default $KANGAROO_REF) at build time only; build/ is git-ignored.
set -e
REF=${REF:-$KANGAROO_REF}
HERE=$(cd "$(dirname "$0")" && pwd)
ROOT=$(cd "$HERE/../.." && pwd)
OUT=$ROOT/build
mkdir -p "$OUT"
FLAGS="-O2 -m64 -mssse3 -fPIC -Wno-unused-result -Wno-write-strings -include cstdint -I$REF"
g++ $FLAGS -shared -o "$OUT/libkgx_ingest.so" "$HERE/kgx_ingest.cpp" "$REF/HashTable.cpp" "$REF/Timer.cpp" \
    "$REF/SECPK1/Int.cpp" "$REF/SECPK1/IntMod.cpp" "$REF/SECPK1/IntGroup.cpp" "$REF/SECPK1/Point.cpp" \
    "$REF/SECPK1/SECP256K1.cpp" "$REF/SECPK1/Random.cpp" -lpthread
echo "built $OUT/libkgx_ingest.so"
