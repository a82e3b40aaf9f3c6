"""CPU: the solver's batch work files (--batch-keys --batch-save / --batch-resume): the argument checks, the batch block's
round trip through kgx_batch_block / kgx_batch_read (libkgx.so, no device needed), its refusals, and the reference program
reading the HEADW part of a batch file as it reads the plain file."""
import os
import struct
import subprocess

import numpy as np
import pytest

from kangaroo_b200 import ecmath as ec
from kangaroo_b200.solver import config_difference, main
from kangaroo_b200.worktool import BatchBlock, batch_block, read_batch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
REF_CPU = os.path.join(ROOT, "oracle", "_ref", "kangaroo_ref_cpu")
CFG = os.path.join(GOLD, "in56_64keys.txt")
START, END, PUBS = ec.parse_config(CFG)


def limbs(v, n=4):
    return struct.pack("<%dQ" % n, *[(v >> (64 * k)) & 0xFFFFFFFFFFFFFFFF for k in range(n)])


def headw(start, end, pub, records, entries=()):
    """a HEADW work file: header, the table (entries: (bucket, x, d) in bucket order), the kangaroo count and the records"""
    out = [struct.pack("<III", 0xFA6A8001, 0, 8), limbs(start), limbs(end), limbs(pub[0]), limbs(pub[1]),
           struct.pack("<Qd", 123456, 1.5)]
    by_bucket = {}
    for h, x, d in entries:
        by_bucket.setdefault(h, []).append(limbs(x, 2) + limbs(d, 2))
    for h in range(1 << 18):
        e = by_bucket.get(h, [])
        out.append(struct.pack("<II", len(e), (len(e) + 3) & ~3) + b"".join(e))
    out.append(struct.pack("<Q", len(records)))
    out += [limbs(x) + limbs(y) + limbs(d) for x, y, d in records]
    return b"".join(out)


def records(keys, targets, seed=1):
    """valid kangaroo records: even index tame at d*G, odd index wild at keys[target] + d*G"""
    rng = np.random.default_rng(seed)
    out = []
    for i, t in enumerate(targets):
        d = int(rng.integers(1, 1 << 55))
        p = ec.mul(d) if i % 2 == 0 else ec.add(keys[int(t)], ec.mul(d))
        out.append((p[0], p[1], d))
    return out


def tame_entries(ds=(11, 22, 33)):
    """table entries of tame DPs d*G: bucket = bits 128..145 of x, the low 128 bits of x, d tagged tame (HashTable::Convert)"""
    out = []
    for d in ds:
        x = ec.mul(d)[0]
        out.append(((x >> 128) & 0x3FFFF, x & ((1 << 128) - 1), d))
    return sorted(out)


def make_batch(tmp_path, n_keys=5, n_walk=10, name="b.work"):
    pubs = PUBS[:n_keys]
    keys = [ec.add(p, ec.neg(ec.mul(START))) for p in pubs]
    targets = np.array([0 if i % 2 == 0 else (i // 2) % n_keys for i in range(n_walk)], dtype=np.uint16)
    plain = headw(START, END, pubs[0], records(keys, targets), tame_entries())
    solved = [i in (1, 3) for i in range(n_keys)]
    privs = [0x1234 + i if s else None for i, s in enumerate(solved)]
    block = BatchBlock(pubs, solved, privs, targets)
    path = tmp_path / name
    path.write_bytes(plain + batch_block(block, len(plain)).tobytes())
    return str(path), plain, block


# ---- the batch block -----------------------------------------------------------------------------------------------------
def test_batch_block_round_trip_from_the_end_of_the_file(tmp_path):
    path, plain, block = make_batch(tmp_path, n_keys=5, n_walk=11)            # 22 bytes of targets: padded to 24
    raw = open(path, "rb").read()
    assert len(raw) - len(plain) == 24 + 5 * 104 + 24 + 16
    offset, magic, version = struct.unpack("<QII", raw[-16:])                  # the footer points back to the block
    assert (offset, magic, version) == (len(plain), 0xBA7C4B01, 1)
    got = read_batch(path)
    assert got.offset == len(plain) and got.n_keys == 5 and got.nb_walk == 11
    assert got.pubs == block.pubs and got.solved == block.solved and got.privs == block.privs
    assert np.array_equal(got.targets, block.targets)
    # no kangaroos (the save a full device table makes) and a file that ends after its table
    p0 = tmp_path / "nowalk.work"
    plain0 = headw(START, END, PUBS[0], [])
    p0.write_bytes(plain0 + batch_block(BatchBlock(PUBS[:2], [True, False], [7, None], []), len(plain0)).tobytes())
    got = read_batch(str(p0))
    assert got.nb_walk == 0 and got.solved == [True, False] and got.privs == [7, None]
    p1 = tmp_path / "tableonly.work"
    p1.write_bytes(plain0[:-8])
    assert read_batch(str(p1)) is None


def test_plain_headw_file_has_no_batch_block(tmp_path):
    p = tmp_path / "plain.work"
    keys = [ec.add(PUBS[0], ec.neg(ec.mul(START)))]
    p.write_bytes(headw(START, END, PUBS[0], records(keys, [0] * 6)))
    assert read_batch(str(p)) is None


def test_truncated_or_damaged_batch_block_is_refused(tmp_path):
    path, plain, _ = make_batch(tmp_path)
    raw = open(path, "rb").read()
    cases = {"cut": raw[:-1], "half": raw[:len(plain) + 100], "footer": raw[:-16] + struct.pack("<QII", len(plain) + 8, 0xBA7C4B01, 1),
             "records": raw[:len(plain) - 96] + raw[len(plain):]}
    bad_target = bytearray(raw)
    bad_target[len(plain) + 24 + 5 * 104 + 2] = 9                           # kangaroo 1's target: 9, with 5 keys
    cases["target"] = bytes(bad_target)
    for name, data in cases.items():
        p = tmp_path / ("bad_%s.work" % name)
        p.write_bytes(data)
        with pytest.raises(ValueError):
            read_batch(str(p))
    with pytest.raises(ValueError, match="not a HEADW"):
        (tmp_path / "junk").write_bytes(b"\0" * 200)
        read_batch(str(tmp_path / "junk"))
    with pytest.raises(ValueError, match="not below n_keys"):
        batch_block(BatchBlock(PUBS[:2], [False, False], [None, None], [0, 2]), 0)


def test_batch_block_round_trip_at_65535_keys(tmp_path):
    """The key limit: 65535 keys with solved flags and private keys at the high indices, an odd number of kangaroos (the
    targets' padding) whose targets cover every key 0..65534, byte patterns that a byte swap or a truncation to 8 bits changes.
    The reader does not check the records or the points, so both are plain patterns here."""
    n_keys, nb_walk = 65535, 2 * 65535 + 3
    rng = np.random.default_rng(12)
    pubs = [(int(a) | (1 << 200), int(b) << 3) for a, b in zip(rng.integers(1, 1 << 62, size=n_keys), rng.integers(1, 1 << 62, size=n_keys))]
    hi = [255, 256, 257, 511, 512, 4095, 4096, 65279, 65280, 65528, 65533, 65534]
    solved = [i in hi or i % 997 == 3 for i in range(n_keys)]
    privs = [(0xA5 << 248) | (i << 16) | 0x5A if s else None for i, s in enumerate(solved)]
    targets = np.empty(nb_walk, dtype=np.uint16)
    targets[0::2] = rng.integers(0, n_keys, size=(nb_walk + 1) // 2)
    targets[1:2 * n_keys:2] = np.arange(n_keys)                           # every key is some wild's target
    targets[-2:] = [0x0100, 65534]
    plain = headw(START, END, PUBS[0], [(i, ~i & 0xFFFF, i) for i in range(nb_walk)])
    block = batch_block(BatchBlock(pubs, solved, privs, targets), len(plain)).tobytes()
    pad = 8 - (2 * nb_walk) % 8
    assert pad == 6 and len(block) == 24 + n_keys * 104 + 2 * nb_walk + pad + 16
    assert block[24 + n_keys * 104 + 2 * nb_walk:][:pad] == b"\0" * pad
    path = tmp_path / "max.work"
    path.write_bytes(plain + block)
    got = read_batch(str(path))
    assert got.n_keys == n_keys and got.nb_walk == nb_walk and got.offset == len(plain)
    assert got.pubs == pubs and got.solved == solved and got.privs == privs
    assert np.array_equal(got.targets, targets) and set(np.unique(got.targets).tolist()) == set(range(n_keys))
    for i in hi:
        assert got.privs[i] == (0xA5 << 248) | (i << 16) | 0x5A and got.pubs[i] == pubs[i]

    # the block of 65536 keys, with every size consistent (the footer, the targets): the reader refuses it on the key count
    raw = plain + block
    at = len(plain) + 24 + n_keys * 104
    big = bytearray(raw[:at] + raw[at - 104:at] + raw[at:])
    big[len(plain) + 8:len(plain) + 12] = struct.pack("<I", n_keys + 1)
    assert len(big) - len(plain) == 24 + (n_keys + 1) * 104 + 2 * nb_walk + pad + 16
    p = tmp_path / "over.work"
    p.write_bytes(bytes(big))
    with pytest.raises(ValueError, match="65536 keys"):
        read_batch(str(p))
    with pytest.raises(ValueError, match="n_keys must be in \\[1, 65535\\]"):
        batch_block(BatchBlock(pubs + [pubs[0]], solved + [False], privs + [None], targets), len(plain))


# ---- flags ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("extra", [["--batch-save", "w.work"], ["--batch-save-interval", "5"], ["--batch-resume", "w.work"]])
def test_batch_flags_need_batch_keys(extra, capsys):
    with pytest.raises(SystemExit) as e:
        main([CFG] + extra)
    assert e.value.code == 2
    assert "need --batch-keys" in capsys.readouterr().err


def test_batch_save_interval_needs_batch_save(capsys):
    with pytest.raises(SystemExit) as e:
        main([CFG, "--batch-keys", "--batch-save-interval", "5"])
    assert e.value.code == 2
    assert "--batch-save-interval needs --batch-save" in capsys.readouterr().err


def test_batch_resume_refuses_a_plain_headw_file(tmp_path, capsys):
    p = tmp_path / "plain.work"
    p.write_bytes(headw(START, END, PUBS[0], []))
    with pytest.raises(SystemExit) as e:
        main(["--batch-keys", "--batch-resume", str(p)])
    assert e.value.code == 2
    assert "plain HEADW work file (no batch block)" in capsys.readouterr().err


def test_batch_resume_refuses_a_damaged_file(tmp_path, capsys):
    path, _, _ = make_batch(tmp_path)
    p = tmp_path / "cut.work"
    p.write_bytes(open(path, "rb").read()[:-5])
    with pytest.raises(SystemExit) as e:
        main(["--batch-keys", "--batch-resume", str(p)])
    assert e.value.code == 2
    assert "cannot resume" in capsys.readouterr().err


def test_batch_resume_refuses_a_config_that_differs(tmp_path, capsys):
    path, _, _ = make_batch(tmp_path, n_keys=5)
    lines = open(CFG).read().split()
    cases = {"key #2 differs": lines[:4] + [lines[5], lines[4], lines[6]],
             "range start": ["%X" % (START + 1)] + lines[1:7],
             "range end": [lines[0], "%X" % (END + 1)] + lines[2:7],
             "lists 4 keys, the file 5": lines[:6],
             "lists 6 keys, the file 5": lines[:8]}
    for want, cfg_lines in cases.items():
        cfg = tmp_path / "cfg.txt"
        cfg.write_text("\n".join(cfg_lines) + "\n")
        with pytest.raises(SystemExit) as e:
            main([str(cfg), "--batch-keys", "--batch-resume", path])
        assert e.value.code == 2
        err = capsys.readouterr().err
        assert "the config does not match" in err and want in err, (want, err)


def test_config_difference_names_the_first():
    pubs = PUBS[:4]
    assert config_difference(START, END, pubs, START, END, pubs) is None
    other = [pubs[0], pubs[2], pubs[1], pubs[3]]
    assert config_difference(START, END, other, START, END, pubs).startswith("key #1 differs")
    assert config_difference(START + 1, END, other, START, END, pubs).startswith("the config's range start")


# ---- the reference reads the HEADW part ----------------------------------------------------------------------------------
@pytest.mark.skipif(not os.path.exists(REF_CPU), reason="oracle/_ref/kangaroo_ref_cpu not built (needs the reference sources at build time)")
def test_reference_reads_the_headw_part_of_a_batch_file(tmp_path):
    """The reference's -winfo and -wcheck read nbLoadedWalk records and ignore what follows: on a batch file they print what
    they print for the same file without its batch block, and -wcheck finds every DP and kangaroo OK."""
    path, plain, _ = make_batch(tmp_path, n_keys=5, n_walk=10)
    # the header key is input key 0: kangaroo 1 (wild, target 0) is key 0's, the other wilds belong to other keys
    p0 = tmp_path / "plain.work"
    p0.write_bytes(plain)
    outs = []
    for f in (path, str(p0)):
        info = subprocess.run([REF_CPU, "-winfo", f], capture_output=True, text=True, timeout=120).stdout
        chk = subprocess.run([REF_CPU, "-t", "1", "-wcheck", f], capture_output=True, text=True, timeout=300).stdout
        outs.append((info.replace(f, "F"), chk.replace(f, "F")))
    assert outs[0] == outs[1], outs
    info, chk = outs[0]
    assert "Kangaroos : 10 " in info and "DP Count  : 3 " in info, info
    assert "[100.000% OK]" in chk, chk
