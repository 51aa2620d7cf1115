"""The steady tick of sym2_kernel (josefine_b200/csrc/sym_fold.cuh) after its per-tick work was cut: the encoder's
in-place run extension (emit_leader / emit_followers only touch the open run while no record closes) and the
AppendEntries id list kept out of local memory (SymMail::id / set_id).  A folding engine, a never-folding engine and
the oracle must agree on replica state, block tables, leader table and Instruction stream (tests/test_sym_fold.py:same)
in the shapes those cuts branch on: every replica count the engine builds, 1..3 blocks per AppendEntries, runs that
close in the middle of a launch (a token off the stride, a tick without a proposal), and pattern windows
(FS_PATTERN_BITS Instructions) that fill in the middle of a launch, at its last tick, or stay open across launches
because the stream is not drained in between."""
import pytest

from tests.stream_cases import _bootstrap, strided_tokens
from tests.test_sym_fold import _emu, _gpu, same, trio


def case_window_edges(make, R, G, n_synth, ticks, drain_every):
    """Launches of jr_run with `n_synth` synthetic proposals per tick (1 + n_synth blocks per AppendEntries; 0 in case_broken_runs), the
    Instruction stream drained every `drain_every` launches: the leader's pattern windows fill at different ticks of
    a launch, and without a drain they carry over into the next launch (whose followers then keep raw FIFOs)."""
    apis = trio(make, G, R, seed=20 + R, chain_capacity=512, fsm_units=2048, fsm_host_records=G * R * 4096)
    for api in apis:
        _bootstrap(api, G, R)
        api.run(100, 100, 10, 1)
    same(apis, chain_ids=0)
    now = 1100
    folded = []
    for k, n in enumerate(ticks):
        for api in apis:
            api.run(now, 100, n, n_synth)
        now += 100 * n
        folded.append(apis[0].fold_count())
        if (k + 1) % drain_every == 0 or k + 1 == len(ticks):
            same(apis, chain_ids=0)
    return folded


def case_broken_runs(make, R, G, ticks=40, launches=4):
    """jr_run_tokens with tokens that leave the stride (the NOTIFY and later the APPLY runs close mid-launch and a new
    one opens), ticks without any proposal (an AppendEntries of 0 blocks, no Notify) and ticks where only some
    groups propose."""
    apis = trio(make, G, R, seed=7 + R, chain_capacity=512, fsm_units=2048, fsm_host_records=G * R * 4096)
    for api in apis:
        _bootstrap(api, G, R)
        api.run(100, 100, 10, 1)
        api.leader_table()
    same(apis, chain_ids=0)
    now, tick = 1100, 0
    folded = []
    for rnd in range(launches):
        toks = strided_tokens(ticks, G, tick)
        for k in range(ticks):
            if (k + rnd) % 11 == 5:
                toks[k] = [0] * G                                   # no proposal at all this tick
            elif (k + 2 * rnd) % 7 == 3:
                toks[k] = [t + 3 if g % 3 == 0 else t for g, t in enumerate(toks[k])]   # off the stride
            elif (k + rnd) % 13 == 8:
                toks[k] = [t if g % 2 else 0 for g, t in enumerate(toks[k])]          # some groups only
        for api in apis:
            api.run_tokens(now, 100, toks)
        now += 100 * ticks
        tick += ticks
        folded.append(apis[0].fold_count())
        same(apis, chain_ids=0)
    return folded


@pytest.mark.parametrize("R", [2, 3, 4, 5, 6, 7, 8])
def test_window_edges_on_device_code(R):
    folded = case_window_edges(_emu, R, 6, 1, [13, 40, 27, 64, 3, 80], 1)
    assert all(f == 6 for f in folded[1:]), folded


@pytest.mark.parametrize("n_synth", [0, 1, 2])
def test_appendentries_sizes_on_device_code(n_synth):
    folded = case_window_edges(_emu, 5, 6, n_synth, [9, 33, 17, 40], 1)
    assert all(f == 6 for f in folded[1:]), folded


@pytest.mark.parametrize("R", [3, 5])
def test_windows_across_launches_on_device_code(R):
    folded = case_window_edges(_emu, R, 6, 1, [21, 50, 33, 64, 7, 40], 3)
    assert all(f == 6 for f in folded[1:]), folded


@pytest.mark.parametrize("R", [2, 5, 8])
def test_broken_runs_on_device_code(R):
    folded = case_broken_runs(_emu, R, 8)
    assert all(f == 8 for f in folded), folded


@pytest.mark.gpu
@pytest.mark.parametrize("R", [2, 3, 4, 5, 6, 7, 8])
def test_window_edges_on_gpu(R):
    folded = case_window_edges(_gpu, R, 1024, 1, [13, 40, 27, 64, 3, 80], 1)
    assert all(f == 1024 for f in folded[1:]), folded


@pytest.mark.gpu
@pytest.mark.parametrize("n_synth", [0, 2])
def test_appendentries_sizes_on_gpu(n_synth):
    folded = case_window_edges(_gpu, 5, 1024, n_synth, [9, 33, 17, 40], 1)
    assert all(f == 1024 for f in folded[1:]), folded


@pytest.mark.gpu
def test_windows_across_launches_on_gpu():
    folded = case_window_edges(_gpu, 5, 1024, 1, [21, 50, 33, 64, 7, 40], 3)
    assert all(f == 1024 for f in folded[1:]), folded


@pytest.mark.gpu
@pytest.mark.parametrize("R", [3, 5])
def test_broken_runs_on_gpu(R):
    folded = case_broken_runs(_gpu, R, 1024)
    assert all(f == 1024 for f in folded), folded
