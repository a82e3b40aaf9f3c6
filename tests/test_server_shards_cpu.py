"""The DP server's sharded table without a GPU: parsing of --devices, and the shards' bucket ranges and work-file piece offsets
against the solver's --dp-table sharded."""
import pytest

from kangaroo_b200 import server
from kangaroo_b200.dist import NBUCKET, owner_of, owner_ranges
from kangaroo_b200.solver import piece_offsets
from tests.server_util import ROOT

CFG = ROOT + "/tests/golden/in56.txt"


def parse(*extra):
    return server.parse_args([CFG, "--dp", "8"] + list(extra))[0]


def refused(capsys, *extra):
    with pytest.raises(SystemExit) as e:
        parse(*extra)
    assert e.value.code == 2
    return capsys.readouterr().err


def test_devices_parsed():
    assert parse("--devices", "0,1,2,3").devices == [0, 1, 2, 3]
    assert parse("--devices", "0,0,0").devices == [0, 0, 0]
    a = parse("--devices", "2")
    assert a.devices == [2] and a.device == 2                  # one entry: the one-GPU server on that GPU
    assert parse("--devices", ",".join(["0"] * 256)).devices == [0] * 256


def test_device_unchanged():
    a = parse()
    assert a.device == 0 and a.devices is None
    a = parse("--device", "3")
    assert a.device == 3 and a.devices is None


def test_devices_refused(capsys):
    assert "not both" in refused(capsys, "--device", "0", "--devices", "0,1")
    assert "empty" in refused(capsys, "--devices", "")
    assert "256" in refused(capsys, "--devices", ",".join(["0"] * 257))
    assert "separated by commas" in refused(capsys, "--devices", "0,,1")
    assert "separated by commas" in refused(capsys, "--devices", "a,b")
    assert "not negative" in refused(capsys, "--devices", "0,-1")


@pytest.mark.parametrize("world", range(1, 9))
def test_shard_ranges_are_the_solvers(world):
    devices = [r % 2 for r in range(world)]
    plan = server.shard_plan(devices)
    assert [d for d, _, _ in plan] == devices
    assert [(lo, hi) for _, lo, hi in plan] == owner_ranges(world)
    assert plan[0][1] == 0 and plan[-1][2] == NBUCKET
    for s, (_, lo, hi) in enumerate(plan):                     # the kernels' owner rule puts each range's ends in its shard
        if lo < hi:
            assert owner_of(lo, world) == s and owner_of(hi - 1, world) == s


@pytest.mark.parametrize("world", range(1, 9))
def test_piece_offsets_are_the_solvers(world):
    plan = server.shard_plan([0] * world)
    counts = [7 * s + 1 for s in range(world)]
    sizes = [8 * (hi - lo) + 32 * c for (_, lo, hi), c in zip(plan, counts)]     # kgx_dptable_piece_bytes
    offs = piece_offsets(sizes)
    assert offs[0] == 156
    assert offs[-1] == 156 + 8 * NBUCKET + 32 * sum(counts)    # where the one table's kangaroo count sits
