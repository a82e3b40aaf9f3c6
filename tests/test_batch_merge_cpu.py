"""CPU: the refusals of `worktool merge` on batch work files that need no device (a plain file mixed in, another key order or
count, another range, conflicting private keys), each leaving no DEST and no DEST.tmp."""
import os

import pytest

from kangaroo_b200 import worktool as wt
from tests.batch_merge_util import CPU_REFUSALS, refusal_inputs


@pytest.mark.parametrize("what", CPU_REFUSALS)
def test_batch_merge_refusals_write_nothing(tmp_path, what):
    inputs, match = refusal_inputs(tmp_path, what)
    dest = str(tmp_path / "dest.work")
    with pytest.raises(ValueError, match=match):
        wt.merge(inputs, dest)
    assert not os.path.exists(dest) and not os.path.exists(dest + ".tmp")
    assert wt.main(["merge"] + inputs + ["-o", dest]) == 2
    assert wt.main(["merge"] + inputs[::-1] + ["-o", dest]) == 2
    assert not os.path.exists(dest) and not os.path.exists(dest + ".tmp")


def test_a_plain_file_first_is_refused_too(tmp_path):
    inputs, _ = refusal_inputs(tmp_path, "plain")
    with pytest.raises(ValueError, match="plain HEADW"):
        wt.merge(inputs[::-1], str(tmp_path / "dest.work"))
