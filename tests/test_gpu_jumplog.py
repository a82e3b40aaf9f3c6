"""The stream kernel's jump-index log over several windows per launch (-m gpu, except the coverage test, which needs no device).
The stream kernel writes one log byte per jump (the jump index; bit 5 the class switch in symmetric mode) and folds the log
into the distances after every LOG_RUNS = 64 runs and after a launch's last run; a DP's distance is rebuilt from the last
fold plus the window's bytes so far.  A wrong fold or rebuild still makes valid-looking walks and DPs, so one engine per case
runs launches of SCHEDULE jumps on the 991,616-kangaroo shape herd and a sample's oracle replay checks every launch bit for
bit.  The resident and cluster kernels keep no log: on the same schedule they show that the schedule and the replay are
right.  LOG_VARIANTS and SYM_LOG_VARIANTS must select every stream instantiation (tests/test_abi_cpu.py)."""
import numpy as np
import pytest

from tests.test_gpu_modes import (KGX_VARS, SHAPE_GRID, SYM_LOOPING, SYM_RP, SYM_RULES, device_sms, herd_start_state,
                                  s128_mod_n, shape_sample, sym_herd_arrays, variant_id)

# 64 fills one window; 65 adds a one-run window after a full one; 129 folds at 64, at 128 and after its last run; 1 follows
# 129, so 63 of its window's bytes are stale ones of the launch before.
SCHEDULE = (64, 65, 129, 1)
# Run positions of a launch at which sample kangaroos must hit DPs: both ends of each replay_window half (0, 31 | 32, 63),
# the first run after a fold inside a launch (64, 128) and the last of a full window (127); in the 65-jump launch, the
# one-run window.
WINDOW_EDGES = {SCHEDULE.index(129): (0, 31, 32, 63, 64, 127, 128), SCHEDULE.index(65): (64,)}
DP_BITS = 10                      # a 129-jump launch: ~125 k DPs in all, ~8 per run position in the sample
MAX_FOUND = 1 << 18
LOG_SAMPLE = 8192                 # strided kangaroos, plus the last 128

# Without KGX_STREAM_G the group size is adaptive: 30 (2 CTAs/SM) or 20 (3 CTAs/SM) on this herd with 132 SMs.
LOG_VARIANTS = [
    {"KGX_MODE": "stream", "KGX_STREAM_G": "128"},          # the benchmarked kernel: warp inverse, 2 CTAs/SM
    {"KGX_MODE": "stream", "KGX_STREAM_CTAS": "2", "KGX_STREAM_INV": "warp"},
    {"KGX_MODE": "stream", "KGX_STREAM_CTAS": "2", "KGX_STREAM_INV": "thread"},
    {"KGX_MODE": "stream", "KGX_STREAM_CTAS": "3", "KGX_STREAM_INV": "warp"},
    {"KGX_MODE": "stream", "KGX_STREAM_CTAS": "3", "KGX_STREAM_INV": "thread"},
    {"KGX_MODE": "stream", "KGX_STREAM_G": "2"},            # CTAs loop over tiles
    {"KGX_MODE": "stream", "KGX_STREAM_G": "130"},          # the longest run stride of the log
    {"KGX_MODE": "resident"},                                # controls: no log
    {"KGX_MODE": "tmem"},
]
SYM_LOG_VARIANTS = [
    {"KGX_MODE": "stream"},
    {"KGX_MODE": "stream", "KGX_STREAM_G": "2"},
    {"KGX_MODE": "stream", "KGX_STREAM_G": "130"},
    {"KGX_MODE": "resident"},                                # control
]


def replay(oracle, x, y, d, table, mask, state=None, rule=None):
    """SCHEDULE replayed on the sample from its start state -> per launch (x, y, d after it, its DPs (x, d, sample index,
    jump of the launch from 1)).  d: biased 128-bit distances, or in symmetric mode d mod n with the state bytes."""
    x, y, d, out = x.copy(), y.copy(), d.copy(), []
    for n_run in SCHEDULE:
        if rule is None:
            dps = oracle.jump_gpu_conv(x, y, d, table, n_run, mask)
        else:
            dps = oracle.jump_sym(x, y, d, state, table, n_run, mask, rule=rule)
        out.append((x.copy(), y.copy(), d.copy(), dps))
    return out


@pytest.fixture(scope="module")
def log_walk(oracle):
    """The non-symmetric shape herd, its sample's start state and the sample's replay."""
    from kangaroo_b200 import random_herd_arrays
    from tests.golden_util import load_cases
    case = [c for c in load_cases() if c["range_power"] == 80][0]
    n = SHAPE_GRID[0] * SHAPE_GRID[1] * 128
    sc, d128 = random_herd_arrays(n, 80, case["width_div2"], np.random.Generator(np.random.PCG64(4545)))
    idx = shape_sample(n, LOG_SAMPLE)
    x, y, d, _ = herd_start_state(oracle, case["key"], sc, d128, idx)
    mask = oracle.dp_mask(DP_BITS)
    return dict(n=n, sc=sc, d128=d128, key=case["key"], wild_offset=case["width_div2"], table=case["table"], mask=mask,
                idx=idx, start=(x, y, d), launches=replay(oracle, x, y, d, case["table"], mask))


@pytest.fixture(scope="module")
def sym_log_walk(oracle):
    """The symmetric shape herd, its sample's start state (class representatives) and the sample's replay under each rule."""
    from tests.golden_util import load_cases
    key =[c for c in load_cases() if c["range_power"] == 80][0]["key"]
    n = SHAPE_GRID[0] * SHAPE_GRID[1] * 128
    sc, d128 = sym_herd_arrays(n, np.random.Generator(np.random.PCG64(4646)))
    idx = shape_sample(n, LOG_SAMPLE)
    x, y, d, flipped = herd_start_state(oracle, key, sc, d128, idx, symmetric=True)
    assert 0 < flipped < len(idx)
    table, mask = oracle.create_jump_table_sym(SYM_RP), oracle.dp_mask(DP_BITS)
    launches = {rule: replay(oracle, x, y, s128_mod_n(d), table, mask, np.full(len(idx), init, dtype=np.uint8), rule)
                for rule, init in SYM_RULES}
    return dict(n=n, sc=sc, d128=d128, key=key, table=table, mask=mask, idx=idx, start=(x, y, d), launches=launches)


def test_sample_dps_sit_at_every_window_edge(log_walk, sym_log_walk):
    """From the replay alone: the sample hits DPs at every run position in WINDOW_EDGES and in every launch, in each engine
    mode, so that a change of seed, dp or sample cannot quietly leave a window edge unchecked."""
    walks = {"non-symmetric": log_walk["launches"]}
    walks.update(sym_log_walk["launches"])
    for name, launches in walks.items():
        hit = [{j - 1 for _, _, _, j in dps} for _, _, _, dps in launches]
        assert all(hit), name
        for launch, runs in WINDOW_EDGES.items():
            assert set(runs) <= hit[launch], (name, SCHEDULE[launch], sorted(set(runs) - hit[launch]))
        assert all(max(hit[launch]) < n_run for launch, n_run in enumerate(SCHEDULE)), name


def run_schedule(env, walk, launches, monkeypatch, rule=None):
    """One engine of variant `env` (symmetric with `rule` unless None) runs SCHEDULE on the walk's herd.  Its sample's start
    state, and after every launch its end state (x, y, biased d or d mod n) and DPs must equal the replay `launches`; no DP
    may come from a padding slot, and no launch may lose one."""
    from kangaroo_b200 import GPUEngine
    for k in KGX_VARS:
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    n, idx = walk["n"], walk["idx"]
    vid = variant_id(env)
    if vid in SYM_LOOPING:            # the tile loop must still happen on this part; the non-symmetric tiles are the same
        assert -(-n // SYM_LOOPING[vid]) > 2 * device_sms(), vid
    eng = GPUEngine(*SHAPE_GRID, 0, MAX_FOUND)
    assert eng.kernel == env["KGX_MODE"]
    if rule is not None:
        eng.SetSymmetry(rule)
    eng.SetParams(walk["mask"], *walk["table"])
    if rule is None:
        eng.SetWildOffset(walk["wild_offset"])
    eng.CreateHerdRaw(walk["sc"], walk["d128"], walk["key"])
    ax, ay, ad = eng.GetKangaroosRaw()
    assert all(np.array_equal(a[idx], b) for a, b in zip((ax, ay, ad), walk["start"]))
    in_sample = set(idx.tolist())
    for launch, (n_run, (wx, wy, wd, dps)) in enumerate(zip(SCHEDULE, launches)):
        eng.set_jumps_per_launch(n_run)
        eng.callKernel()
        found = eng.Launch(relaunch=False)
        assert len(found) == eng.lastFound <= MAX_FOUND, (launch, n_run)
        ax, ay, ad = eng.GetKangaroosRaw()
        gd = ad[idx] if rule is None else s128_mod_n(ad[idx])
        assert np.array_equal(ax[idx], wx) and np.array_equal(ay[idx], wy) and np.array_equal(gd, wd), (launch, n_run)
        assert found and max(it.kIdx for it in found) < n, (launch, n_run)
        got = sorted((it.x, it.d, it.kIdx) for it in found if it.kIdx in in_sample)
        exp = sorted((x, d if rule else eng._unbias(d, int(idx[k])), int(idx[k])) for x, d, k, _ in dps)
        assert got == exp, (launch, n_run)
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize("env", LOG_VARIANTS, ids=[variant_id(v) for v in LOG_VARIANTS])
def test_jump_log_windows_match_oracle(env, log_walk, monkeypatch):
    run_schedule(env, log_walk, log_walk["launches"], monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("rule", [r for r, _ in SYM_RULES])
@pytest.mark.parametrize("env", SYM_LOG_VARIANTS, ids=[variant_id(v) for v in SYM_LOG_VARIANTS])
def test_symmetric_jump_log_windows_match_oracle(env, rule, sym_log_walk, monkeypatch):
    """The folds inside a launch and the DPs rebuilt after them replay the class switches too."""
    run_schedule(env, sym_log_walk, sym_log_walk["launches"][rule], monkeypatch, rule)
