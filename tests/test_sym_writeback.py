"""The followers' write-back row cache of the symmetric-group fold (josefine_b200/csrc/sym_fold.cuh, DESIGN.md §3b).
A row the follower lane appends stays in the cache until a later append evicts it or the launch ends.  It is then
dropped if it lies below min(follower commit, leader commit) - margin, which never exceeds the floor the launch's fused
truncation ends with; otherwise it is stored to every follower's table.  The fused truncation then blanks the
followers' tables only up to the highest row they can hold, which relies on one invariant: no replica holds a row above
its max key.

After every launch the folding engine must equal the never-folding engine and the oracle on the whole table window
(ids above every head included), the checkpoint bytes and everything same() compares: at margins that drop nearly every
row, at one where every eviction is written back, without the fused truncation, with the cache wrapping within a few
ticks, and with aborts after rows were dropped.  The invariant itself is checked on the checkpoint after every launch."""
import numpy as np
import pytest

from tests import test_sym_fold
from tests.stream_cases import _bootstrap
from tests.test_sym_abort import ABSENT, _segments, case_proposal_aborts, check_launch, checkpoint, trio
from tests.test_sym_fold import _emu, _gpu


def no_row_above_max_key(api):
    """Every replica's window [floor, floor + chain_capacity): each id above the replica's max key is absent."""
    ck = checkpoint(api)
    _, Gp, _, rows = _segments(api)
    G, R, cap = api.n_groups, api.n_replicas, api.cfg.chain_capacity
    mk = ck["mk"].view(np.uint32).reshape(R, Gp)[:, :G].astype(np.int64)
    tb = ck["tb"].view(np.uint32)[:G].astype(np.int64)
    cnext = ck["cnext"].view(np.uint32).reshape(rows, R, Gp)[:, :, :G]
    off = (np.arange(rows).reshape(rows, 1, 1) - tb.reshape(1, 1, G)) % rows   # slot s holds id floor + off
    above = (off < cap) & (tb.reshape(1, 1, G) + off > mk.reshape(1, R, G))
    bad = above & (cnext != ABSENT)
    assert not bad.any(), f"rows above the max key are present: (slot, replica, group) {np.argwhere(bad)[:5].tolist()}"


def check(apis, **kw):
    check_launch(apis, **kw)
    for api in apis[:2]:
        no_row_above_max_key(api)


def case_margins(make, G, R, margin, n_synth, launches=4, ticks=33):
    """Steady launches of `ticks` ticks with 1 + n_synth proposals each, ending with jr_truncate(margin) (fused in the
    fold) or, for margin None, without the fused truncation (then an explicit jr_truncate keeps the window moving)."""
    apis = trio(make, G, R, seed=40 + R, chain_capacity=256, fsm_units=256, fsm_host_records=G * R * 256, mailbox_units=64)
    for api in apis:
        _bootstrap(api, G, R, node=2 if R > 2 else 1)
        api.run(100, 100, 12, 1)
        api.leader_table()
        api.set_auto_truncate(margin)
    now = 1300
    for _ in range(launches):
        for api in apis:
            api.run(now, 100, ticks, n_synth)
            if margin is None:
                api.truncate(4)
        now += 100 * ticks
        check(apis, aborted=[], log={})                      # (the host build: no lane aborted, SA_DROPPED included)
    floors = [int(apis[0].query(g, 1).chain_floor) for g in range(G)]
    assert min(floors) > 40, min(floors)                     # the window really moved
    return apis


# margins 0, 1 and 8 drop nearly every row the cache evicts; at 40 (more than the 16 entries) every eviction is written
# back; None: no fused truncation, nothing is dropped.  2 and 3 proposals per tick wrap the cache every 5 to 8 ticks.
@pytest.mark.parametrize("R,margin,n_synth", [(5, 0, 1), (5, 1, 1), (5, 8, 1), (5, 40, 1), (5, None, 1), (5, 8, 2),
                                              (2, 8, 1), (2, 0, 2), (3, 1, 2), (3, 40, 2), (7, 8, 1), (7, None, 2)])
def test_writeback_margins_on_device_code(R, margin, n_synth):
    case_margins(_emu, 70, R, margin, n_synth)


def test_aborts_after_drops_on_device_code():
    """The leader lane aborts at ticks 0, 1, n/2, n-2 and n-1 of 40, one block per tick and margin 1: from about tick 17
    on, the follower lane has dropped rows that the launch, now aborted, will not truncate.  Nothing may be left of
    them; step_kernel re-runs the group from its untouched planes."""
    apis = case_proposal_aborts(_emu, 150, 5, lead=2, n=40, rounds=2, auto_truncate=1, cfg_over=dict(chain_capacity=128))
    for api in apis[:2]:
        no_row_above_max_key(api)


@pytest.mark.parametrize("seed", range(4))
def test_no_row_above_max_key_in_random_scripts_on_device_code(seed, monkeypatch):
    """The invariant the narrowed truncation relies on, after every launch of the fold's random scripts (silenced and
    revived nodes, elections, compaction, explicit and fused truncation, aborts)."""
    same = test_sym_fold.same

    def same_and_invariant(apis, **kw):
        same(apis, **kw)
        for api in apis[:2]:
            no_row_above_max_key(api)

    monkeypatch.setattr(test_sym_fold, "same", same_and_invariant)
    folded_any, _ = test_sym_fold._random_script(_emu, seed, chain_capacity=64)
    assert folded_any


@pytest.mark.gpu
@pytest.mark.parametrize("R,margin,n_synth", [(5, 1, 1), (5, 8, 2), (5, 40, 1), (7, None, 1)])
def test_writeback_margins_on_gpu(R, margin, n_synth):
    case_margins(_gpu, 2112, R, margin, n_synth, launches=3)


@pytest.mark.gpu
def test_aborts_after_drops_on_gpu():
    case_proposal_aborts(_gpu, 4161, 5, lead=2, n=40, rounds=1, every=8, auto_truncate=1, cfg_over=dict(chain_capacity=128))
