"""The symmetric-group fold's entry checks (sym_check_kernel running sym_enter, josefine_b200/csrc/sym_fold.cuh): one engine
whose groups each break exactly one entry condition while the rest stay symmetric.  The broken groups must be left to
step_kernel and every other group must fold; afterwards everything equals an engine that never folds, restored from the
same checkpoint.  The conditions are set by editing a checkpoint (jr_engine_save), so the C++ restatement, which has no
checkpoints, does not take part; tests/test_sym_fold.py compares the fold with it scenario by scenario."""
import numpy as np
import pytest

from josefine_b200 import abi
from tests.stream_cases import _bootstrap
from tests.test_sym_fold import CAP, same

G, R = 20, 5
CFG = dict(seed=21, chain_capacity=64, fsm_units=256, heartbeat_ms=100, mailbox_units=64, flags=CAP)
TICKS, N_SYNTH = 8, 1
QUEUE_CAP = 4                                   # JR_CLIENT_QUEUE_CAP


class Checkpoint:
    """Numpy views of the state planes inside a jr_engine_save blob (segment order of save_segments, engine.cu)."""

    def __init__(self, blob):
        self.buf = bytearray(blob)
        Gp = -(-G // 32) * 32
        self.Gp, plane = Gp, R * Gp
        rows = 1
        while rows < CFG["chain_capacity"]:
            rows *= 2
        self.rows = rows
        U, F = CFG["mailbox_units"], CFG["fsm_units"]
        segs = [("p0", plane * 4, np.uint32), ("p1", plane * 4, np.uint32), ("p2", plane * 4, np.uint32),
                ("p3", plane * 4, np.uint32), ("pr", plane * ((R + 3) // 4) * 4, np.uint32), ("mk", plane, np.uint32),
                ("qt", plane * QUEUE_CAP * 4, np.uint32), ("dg", plane * 4, np.uint32), ("cn", plane * 2, np.uint32),
                ("cnext", plane * rows, np.uint32), ("ctok", plane * rows, np.uint64),
                ("ob0", plane * U * 4, np.uint32), ("ob1", plane * U * 4, np.uint32),
                ("oc0", plane, np.uint32), ("oc1", plane, np.uint32), ("fs", plane * 2 * F * 4, np.uint32),
                ("fc", plane * 2, np.uint32), ("tb", Gp, np.uint32), ("route", G, np.uint32)]
        total = sum(n * np.dtype(t).itemsize for _, n, t in segs)
        at = len(self.buf) - total                # the header's size
        self.cur = int(np.frombuffer(self.buf, np.uint32, 1, at - 16)[0])
        for name, n, t in segs:
            setattr(self, name, np.frombuffer(self.buf, t, n, at))
            at += n * np.dtype(t).itemsize
        assert at == len(self.buf)

    def rg(self, r, g):
        return r * self.Gp + g

    def unit(self, buf, k, r, g):                 # outbox unit k of replica r: a writable uint4 view
        ob = self.ob0 if buf == 0 else self.ob1
        i = ((k * R + r) * self.Gp + g) * 4
        return ob[i:i + 4]

    def count(self, buf, r, g):
        return int((self.oc0 if buf == 0 else self.oc1)[self.rg(r, g)])

    def row(self, r, bid, g):
        return (bid & (self.rows - 1)) * R * self.Gp + self.rg(r, g)


def _quad(a, r, g, ck):
    i = ck.rg(r, g) * 4
    return a[i:i + 4]


# Replica 0 leads every group (node 1 won the bootstrap election); 1 is the lowest follower, whose table stands for all.
def faulted(ck, g): _quad(ck.p2, 3, g, ck)[3] |= 5 << 8
def silenced(ck, g): _quad(ck.p2, 2, g, ck)[3] |= 1 << 27
def queued_request(ck, g): _quad(ck.p2, 2, g, ck)[3] |= 1 << 24
def two_leaders(ck, g): _quad(ck.p2, 3, g, ck)[3] = (_quad(ck.p2, 3, g, ck)[3] & ~np.uint32(255)) | abi.ROLE_LEADER
def follower_term(ck, g): _quad(ck.p0, 2, g, ck)[0] += 1
def follower_head(ck, g): _quad(ck.p2, 4, g, ck)[0] -= 1
def follower_commit(ck, g): _quad(ck.p2, 2, g, ck)[1] -= 1
def follower_max_key(ck, g): ck.mk[ck.rg(3, g)] += 1
def progress_entry(ck, g): _quad(ck.pr, 0, g, ck)[2] -= 1            # the leader's entry for replica 2


def follower_row(ck, g):                                            # a token inside [flo, fmaxkey] in one follower only
    top = int(ck.mk[ck.rg(3, g)])
    ck.ctok[ck.row(3, top, g)] ^= np.uint64(1)


def leader_mail(ck, g):                                             # an AppendEntries block that is not the leader's row
    buf = 1 - ck.cur
    for k in range(ck.count(buf, 0, g)):
        h = ck.unit(buf, k, 0, g)
        if h[0] & 15 == abi.CMD_APPEND_ENTRIES and not (h[0] >> 4) & 1:
            assert (h[0] >> 8) & 255, "the AppendEntries in flight carries no block"
            ck.unit(buf, int(h[3]), 0, g)[2] ^= 1
            return
    raise AssertionError("no AppendEntries in flight")


def follower_mail(ck, g):                                           # one follower answers differently from the others
    buf = 1 - ck.cur
    assert ck.count(buf, 3, g) > 0
    ck.unit(buf, 0, 3, g)[3] += 1


def election_timer(ck, g):                                          # could fire before the first heartbeat arrives
    b = _quad(ck.p1, 4, g, ck)
    b[0], b[1], b[2] = 0, 0, 1


def no_room(ck, g):                                                 # the launch's appends would leave the window
    top = int(ck.mk[ck.rg(0, g)])
    ck.tb[g] = top + TICKS * (1 + N_SYNTH) + 2 - CFG["chain_capacity"]


BREAKS = [faulted, silenced, queued_request, two_leaders, follower_term, follower_head, follower_commit, follower_max_key,
          progress_entry, follower_row, leader_mail, follower_mail, election_timer, no_room]


def heartbeat_in_flight(ck, g=0):
    buf = 1 - ck.cur
    return ck.count(buf, 0, g) > 0 and ck.unit(buf, 0, 0, g)[0] & 15 == abi.CMD_HEARTBEAT


def case_entry_checks(make, monkeypatch):
    fold = make(G, R, **CFG)
    monkeypatch.setenv("JR_NO_FOLD", "1")
    plain = make(G, R, **CFG)                                       # same configuration (a checkpoint fits both), never folds
    monkeypatch.delenv("JR_NO_FOLD")
    _bootstrap(fold, G, R)
    now = 100
    for ticks in (16, 16, 16, 16):
        fold.run(now, 100, ticks, N_SYNTH)
        fold.truncate(6)
        now += 100 * ticks
    assert fold.fold_count() == G
    for _ in range(3):                                              # the election-timer check needs a launch that starts
        ck = Checkpoint(fold.save())                                # without a Heartbeat in flight
        if not heartbeat_in_flight(ck):
            break
        fold.run(now, 100, 5, N_SYNTH)
        now += 500
    else:
        raise AssertionError("a Heartbeat is always in flight")
    assert fold.fold_count() == G
    fold.drain_fsm(cap=1 << 20)
    ck = Checkpoint(fold.save())
    assert int(ck.tb[len(BREAKS)]) > 0
    for g, brk in enumerate(BREAKS, start=1):
        brk(ck, g)
    for api in (fold, plain):
        api.restore(bytes(ck.buf))
        api.run(now, 100, TICKS, N_SYNTH)
    assert fold.fold_count() == G - len(BREAKS)
    assert plain.fold_count() == 0
    same([fold, plain], chain_ids=0)
    now += 100 * TICKS
    for api in (fold, plain):
        api.run(now, 100, TICKS, N_SYNTH)
    same([fold, plain], chain_ids=0)


def _emu(g, r, **kw):
    from tests.emu.emu import EmuEngine
    return EmuEngine.create(g, r, **kw)


def _gpu(g, r, **kw):
    from josefine_b200 import RaftEngine
    return RaftEngine.create(g, r, **kw)


@pytest.mark.parametrize("one_lane", [False, True])
def test_entry_checks_on_device_code(one_lane, monkeypatch):
    if one_lane:
        monkeypatch.setenv("JR_SYM_ONE_LANE", "1")
    case_entry_checks(_emu, monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("one_lane", [False, True])
def test_entry_checks_on_gpu(one_lane, monkeypatch):
    if one_lane:
        monkeypatch.setenv("JR_SYM_ONE_LANE", "1")
    case_entry_checks(_gpu, monkeypatch)
