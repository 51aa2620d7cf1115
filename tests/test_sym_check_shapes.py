"""The fold's entry checks (sym_check_kernel, josefine_b200/csrc/sym_fold.cuh) run one CTA per 32 groups with one warp per
replica.  These cases cover what that mapping adds: a last CTA with lanes past the last group (G = 1, 31, 33, 95), CTAs
of 2, 3, 5 and 8 warps, and leaders on every replica index (group g elects node g % R + 1), so that every warp of a
CTA plays the leader for some lanes and a follower for the others.  After the groups reach the steady state every one
of them must fold, and state, block tables, leader table and Instruction stream must equal an engine that never folds."""
import ctypes as C

import numpy as np
import pytest

from josefine_b200 import abi, Command
from tests import parity
from tests.test_sym_fold import CAP, same


def scattered_bootstrap(api, G, R):
    inj = []
    for g in range(G):
        node = g % R + 1
        inj.append(Command.timeout(g, node))
        for v in [v for v in range(1, R + 1) if v != node][:R // 2]:
            inj.append(Command.vote_response(g, node, 1, v, True))
    api.step(0, flags=0, inject=inj)


def steady_pair(make, G, R, ticks, **over):
    cfg = dict(seed=G * 16 + R, chain_capacity=128, fsm_units=64, heartbeat_ms=100, **over)
    fold = make(G, R, flags=CAP, **cfg)
    plain = make(G, R, flags=CAP | abi.F_NO_SYMMETRIC_FOLD, **cfg)
    now = 100
    for api in (fold, plain):
        scattered_bootstrap(api, G, R)
    for _ in range(2):                      # elections settle, the followers catch up: from here on every group folds
        for api in (fold, plain):
            api.run(now, 100, ticks, 1)
            api.truncate(6)
        now += 100 * ticks
    return fold, plain, now


def case_shapes(make, G, R, launches=3, ticks=16):
    fold, plain, now = steady_pair(make, G, R, ticks)
    assert {e[1] for e in fold.leader_table()} == set(range(1, min(G, R) + 1))
    same([fold, plain])
    for _ in range(launches):
        for api in (fold, plain):
            api.run(now, 100, ticks, 1)
            api.truncate(6)
        now += 100 * ticks
        assert fold.fold_count() == G and plain.fold_count() == 0
        same([fold, plain])


def _emu(g, r, **kw):
    from tests.emu.emu import EmuEngine
    return EmuEngine.create(g, r, **kw)


def _gpu(g, r, **kw):
    from josefine_b200 import RaftEngine
    return RaftEngine.create(g, r, **kw)


@pytest.mark.parametrize("G", [1, 31, 33, 95])
@pytest.mark.parametrize("R", [2, 3, 5, 8])
def test_entry_check_shapes_on_device_code(G, R):
    case_shapes(_emu, G, R)


@pytest.mark.gpu
@pytest.mark.parametrize("G", [1, 31, 33, 95])
@pytest.mark.parametrize("R", [2, 3, 5, 8])
def test_entry_check_shapes_on_gpu(G, R):
    case_shapes(_gpu, G, R)


def _drain_bytes(api, cap):
    buf = (abi.FsmInstr * cap)()
    n = C.c_size_t(0)
    assert api._fn("drain_fsm")(api._h, buf, C.c_size_t(cap), C.byref(n)) == abi.OK
    return np.frombuffer(buf, np.uint8, n.value * C.sizeof(abi.FsmInstr)).copy()


@pytest.mark.gpu
def test_scattered_leaders_full_size_on_gpu():
    """65,536 x 5 with leaders on every replica index: every group folds, and the whole Instruction stream, the state and
    leader table digests, and the rows of a sample of groups equal the never-folding engine's."""
    G, R, ticks = 65536, 5, 8
    fold, plain, now = steady_pair(_gpu, G, R, ticks, fsm_host_records=G * R * 8)
    cap = G * (R + 1) * ticks * 2
    for api in (fold, plain):
        api.discard_fsm(strict=False)          # the elections' records: not compared here
    for _ in range(2):
        for api in (fold, plain):
            api.run(now, 100, ticks, 1)
            api.truncate(6)
        now += 100 * ticks
        assert fold.fold_count() == G and plain.fold_count() == 0
        a, b = _drain_bytes(fold, cap), _drain_bytes(plain, cap)
        assert len(a) > 0 and np.array_equal(a, b), "Instruction streams differ"
        assert fold.state_digest() == plain.state_digest()
        assert fold.leader_table() == plain.leader_table()
        assert fold.fault_count() == plain.fault_count() == 0
        parity.compare_states(fold, plain, groups=range(0, G, 331), chain_ids=48)
