"""Replica verification (jr_verify_groups): the device's report and findings equal the Python restatement of the rules
(josefine_b200/verify.py) over the engine's state and over the oracle's, clean runs are clean, constructed violations
are found and nothing else is, and the call changes nothing.  Checked on the device code built for the host and on the
GPU."""
import ctypes as C
import os
import subprocess

import pytest

from josefine_b200 import abi, Command, RaftError, verify
from tests import parity, test_sym_fold
from tests.stream_cases import _bootstrap
from tests.test_bulk_restart import _history
from tests.test_sym_fold import trio

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _oracle(g, r, **kw):
    from oracle.restated import RestatedCluster
    return RestatedCluster.create(g, r, n_threads=16 if g >= 1024 else 1, **kw)


def _emu(g, r, **kw):
    from tests.emu.emu import EmuEngine
    return EmuEngine.create(g, r, **kw)


def _gpu(g, r, **kw):
    from josefine_b200 import RaftEngine
    return RaftEngine.create(g, r, **kw)


def _t(res):
    rep, findings = res
    return rep.as_tuple(), [f.as_tuple() for f in findings]


def agree(eng, ora=None, groups=None):
    """jr_verify_groups on the engine == verify.py over the engine's state (== verify.py over the oracle's state)."""
    dev = _t(eng.verify_groups(groups))
    assert dev == _t(verify.verify_groups(eng, groups))
    if ora is not None:
        assert not hasattr(ora._lib, "jro_verify_groups")   # the oracle's verify_groups IS the restatement
        assert dev == _t(ora.verify_groups(groups))
    return dev


def found(res):
    """{(group, kind, node, id)} of a verify result."""
    return {(f[0], f[1], f[2], f[5]) for f in res[1]}


# ---- 1. device == restatement ----------------------------------------------------------------------------------------

def case_history(make, R, monkeypatch):
    """Elections, proposals, truncation, compact and a dead branch (tests/test_bulk_restart._history), checked after
    every step on the engine and on the oracle."""
    step = parity.Pair.step
    checks = []

    def checked_step(self, now, **kw):
        r = step(self, now, **kw)
        checks.append(agree(self.b, self.a))
        return r

    monkeypatch.setattr(parity.Pair, "step", checked_step)
    p, _, _ = _history(make, 6, R, seed=3)
    agree(p.b, p.a)
    assert len(checks) > 15 and all(rep[1] > 0 for rep, _ in checks)


def case_random_script(make, seed, monkeypatch, **kw):
    """test_sym_fold's randomised scripts (faults, silenced leaders, truncation, compaction, fold entry and exit), with the
    check run on the folding engine, the non-folding engine and the oracle after every launch."""
    same = test_sym_fold.same
    seen = []

    def same_and_verified(apis, **skw):
        same(apis, **skw)
        res = agree(apis[0], apis[2])
        assert _t(apis[1].verify_groups()) == res
        seen.append(res)

    monkeypatch.setattr(test_sym_fold, "same", same_and_verified)
    test_sym_fold._random_script(make, seed, **kw)
    assert seen
    return seen


@pytest.mark.parametrize("R", [3, 5, 7])
def test_history_on_device_code(R, monkeypatch):
    case_history(_emu, R, monkeypatch)


@pytest.mark.parametrize("seed", range(8))
def test_random_scripts_on_device_code(seed, monkeypatch):
    case_random_script(_emu, seed, monkeypatch)


# ---- 2. clean runs are clean -----------------------------------------------------------------------------------------

def case_steady_clean(make, R, G=16):
    apis = trio(make, G, R, seed=R, chain_capacity=128, fsm_units=256)
    for api in apis:
        _bootstrap(api, G, R)
        api.set_auto_truncate(6 if R % 2 else None)
    now = 100
    for _ in range(3):
        for api in apis:
            api.run(now, 100, 24, 1)
        now += 2400
        test_sym_fold.same(apis, chain_ids=0)
        want = ((G, G * R, 0, 0, 0, 0, 0, 0), [])
        for api in apis:
            assert _t(api.verify_groups()) == want
        assert agree(apis[0], apis[2]) == want
    assert apis[0].fold_count() == G and apis[1].fold_count() == 0


@pytest.mark.parametrize("R", [2, 3, 4, 5, 6, 7, 8])
def test_steady_state_is_clean_on_device_code(R):
    case_steady_clean(_emu, R)


# ---- 3. constructed violations ---------------------------------------------------------------------------------------

def _pair(make, G, R, **cfg):
    cfg = dict(dict(seed=5, chain_capacity=64), **cfg)
    eng, ora = make(G, R, **cfg), _oracle(G, R, **cfg)
    for api in (eng, ora):
        _bootstrap(api, G, R)
        api.run(100, 100, 16, 1)
    return eng, ora


def _export(eng, g, n):
    (commit, ck, blocks), = eng.chain_export_many([(g, n)])
    return commit, ck, {b[0]: b for b in blocks}


def case_restored_chains(make, G=8, R=5):
    """Replicas restarted from doctored exports: a token changed below the commit, the commit block missing, a next that
    skips to an absent id, a self-loop."""
    eng, ora = _pair(make, G, R)
    assert agree(eng, ora)[1] == []
    expect, chains = set(), []
    for g in (1, 4):                                         # one token changed two blocks below the commit
        c, ck, b = _export(eng, g, 2)
        b[c - 2] = (c - 2, b[c - 2][1], b[c - 2][2] ^ 0x5A5A)
        chains.append((g, 2, sorted(b.values()), c, ck))
        expect.add((g, abi.VERIFY_DIVERGED, 2, c - 2))
    for g in (2, 4):                                         # the commit block left out
        c, ck, b = _export(eng, g, 3)
        del b[c]
        chains.append((g, 3, sorted(b.values()), c, ck))
        expect.add((g, abi.VERIFY_COMMIT_ABSENT, 3, c))
    c, ck, b = _export(eng, 5, 4)                            # the commit's next skips to an id that is not there
    del b[c - 3]
    b[c] = (c, c - 3, b[c][2])
    chains.append((5, 4, sorted(b.values()), c, ck))
    expect.add((5, abi.VERIFY_CHAIN_BROKEN, 4, c - 3))
    c, ck, b = _export(eng, 6, 5)                            # a block that names itself: the walk must still end
    b[c - 1] = (c - 1, c - 1, b[c - 1][2])
    chains.append((6, 5, sorted(b.values()), c, ck))
    expect.add((6, abi.VERIFY_CHAIN_BROKEN, 5, c - 1))
    for api in (eng, ora):
        api.node_restart_many(9000, chains)
    res = agree(eng, ora)
    assert found(res) == expect
    rep = res[0]
    assert rep[3:] == (0, 2, 2, 2, 0) and rep[1] == G * R
    for f in res[1]:
        assert f[3] == 1 and f[4] == 1 << (f[2] - 1) and f[6] == 0   # ref = the leader; the restarted replica's term 0


def case_forged_extend(make, G=6, R=3):
    """AppendEntries from the current leader that rewrites a block the follower already committed: the reference's
    Chain::extend overwrites it (chain.rs:178-192), and the check reports the follower."""
    eng, ora = _pair(make, G, R)
    expect, inj = set(), []
    for g in (0, 3):
        st = eng.query(g, 3)
        c = int(st.commit)
        x = c - 1
        (blk,) = eng.chain_read(g, 3, x, 1)
        inj.append(Command.append_entries(g, 3, term=int(st.current_term), leader_id=1, blocks=[(x, blk[1], 0xF0F0)]))
        expect.add((g, abi.VERIFY_DIVERGED, 3, x))
    for api in (eng, ora):
        api.step(9000, flags=0, inject=inj)
    for g, _, _, x in expect:
        assert ora.query(g, 3).fault == 0 and ora.chain_read(g, 3, x, 1)[0][2] == 0xF0F0   # the oracle accepted it
        assert int(ora.query(g, 3).commit) > x
    assert found(agree(eng, ora)) == expect


def case_two_leaders_and_skips(make, G=5, R=3):
    """Node 2 of a led group restarted (term 0), then Timeout and one granted VoteResponse: two leaders in term 1.
    Then it faults on its first append, another group loses a follower: both are skipped, and the conflict is gone."""
    eng, ora = _pair(make, G, R)
    for api in (eng, ora):
        api.node_restart_many(9000, [(g, 2, None, 0, None) for g in (1, 3)])
        api.step(9000, flags=0, inject=[m for g in (1, 3) for m in (Command.timeout(g, 2),
                                                                   Command.vote_response(g, 2, 1, 3, True))])
    res = agree(eng, ora)
    assert res[1] == [(g, abi.VERIFY_LEADER_CONFLICT, 0, 1, 0b011, 0, 1) for g in (1, 3)]
    assert res[0] == (G, G * R, 0, 0, 0, 0, 0, 2)
    for api in (eng, ora):
        api.step(9010, flags=0, inject=[Command.client_request(1, 2, token=99)])
        api.set_alive(4, 3, False)
    assert eng.query(1, 2).fault == abi.FAULT_APPEND_ID_NOT_GT_HEAD
    res = agree(eng, ora)
    assert res == ((G, G * R - 2, 2, 0, 0, 0, 0, 1), [(3, abi.VERIFY_LEADER_CONFLICT, 0, 1, 0b011, 0, 1)])


def case_below_floor(make, G=4, R=3):
    """A replica silenced while its group's floor moves past its commit, then revived: BELOW_FLOOR, not a violation."""
    eng, ora = _pair(make, G, R)
    for api in (eng, ora):
        api.set_alive(2, 3, False)
        api.run(2000, 100, 20, 1)
        api.truncate(2)
        api.set_alive(2, 3, True)
    c = int(eng.query(2, 3).commit)
    assert c < int(eng.query(2, 3).chain_floor)
    res = agree(eng, ora)
    assert found(res) == {(2, abi.VERIFY_BELOW_FLOOR, 3, c)}


def test_restored_chains_on_device_code():
    case_restored_chains(_emu)


def test_forged_extend_on_device_code():
    case_forged_extend(_emu)


def test_two_leaders_and_skips_on_device_code():
    case_two_leaders_and_skips(_emu)


def test_below_floor_on_device_code():
    case_below_floor(_emu)


# ---- 4. read-only, 5. arguments --------------------------------------------------------------------------------------

def case_read_only(make, G=12, R=5):
    """Digest and checkpoint bytes unchanged by the call (with findings to pack); a fused run after it equals an engine
    that never verified; outstanding Instruction batches are unaffected."""
    cfg = dict(seed=7, chain_capacity=128, flags=abi.F_CAPTURE_FSM, fsm_units=128)
    a, b = make(G, R, **cfg), make(G, R, **cfg)
    for api in (a, b):
        _bootstrap(api, G, R)
        api.run(100, 100, 16, 1)
        c, ck, blocks = api.chain_export_many([(3, 2)])[0]
        blocks = [(i, n, t ^ 1) if i == c - 1 else (i, n, t) for i, n, t in blocks]
        api.node_restart_many(2000, [(3, 2, blocks, c, ck)])
    digest, blob = a.state_digest(), a.save()
    res = _t(a.verify_groups())
    assert found(res) == {(3, abi.VERIFY_DIVERGED, 2, c - 1)}
    assert a.state_digest() == digest and a.save() == blob
    # with an Instruction batch outstanding (the run's records are still undrained)
    assert a._fn("fsm_records_async")(a._h) == abi.OK
    assert _t(a.verify_groups([3, 5])) == ((2, 2 * R, 0, 0, 0, 0, 1, 0), res[1])
    ptr, batch = C.POINTER(abi.FsmRecord)(), abi.FsmBatch()
    assert a._fn("fsm_records_wait")(a._h, C.byref(ptr), C.byref(batch)) == abi.OK
    recs_a = [bytes(abi.FsmRecord.from_buffer_copy(ptr[i])) for i in range(batch.n_records)]
    recs_b = [bytes(r) for r in b.fsm_records()[0]]
    assert recs_a == recs_b and batch.n_records > 0
    for api in (a, b):
        api.run(2800, 100, 24, 1)
    test_sym_fold.same([a, b], chain_ids=64)   # state, block tables, digest, leader table and Instruction stream


def case_arguments(make, G=10, R=3):
    eng, ora = _pair(make, G, R)
    for api in (eng, ora):
        api.set_alive(7, 2, False)
        c, ck, blocks = api.chain_export_many([(2, 3)])[0]
        api.node_restart_many(9000, [(2, 3, [b for b in blocks if b[0] != c], c, ck)])
        c, ck, blocks = api.chain_export_many([(6, 2)])[0]
        api.node_restart_many(9000, [(6, 2, [(i, n, t + (i == c)) for i, n, t in blocks], c, ck)])
    full = agree(eng, ora)
    assert len(full[1]) == 2
    fn = eng._fn("verify_groups")
    digest = eng.state_digest()
    rep, need = abi.VerifyReport(), C.c_size_t(0)
    for bad in ([G], [1, 1], [0, G + 5], [3, 4, 3]):
        arr = (C.c_uint32 * len(bad))(*bad)
        assert fn(eng._h, arr, len(bad), C.byref(rep), None, 0, C.byref(need)) == abi.E_INVAL, bad
        for api in (eng, ora):
            with pytest.raises(RaftError):
                api.verify_groups(bad)
    assert fn(eng._h, None, 3, C.byref(rep), None, 0, C.byref(need)) == abi.E_INVAL
    assert eng.state_digest() == digest
    # capacity: no buffer, one too few, exactly enough
    out = (abi.VerifyFinding * 2)()
    for buf, cap in ((None, 0), (out, 1)):
        rep, need = abi.VerifyReport(), C.c_size_t(0)
        assert fn(eng._h, None, 0, C.byref(rep), buf, cap, C.byref(need)) == abi.E_CAPACITY
        assert need.value == 2 and rep.as_tuple() == full[0]
    assert fn(eng._h, None, 0, C.byref(rep), out, 2, C.byref(need)) == abi.OK
    assert [f.as_tuple() for f in out] == full[1]
    # an empty list checks nothing; a subset (in any order) gives the full check's findings for those groups
    assert _t(eng.verify_groups([])) == ((0,) + (0,) * 7, [])
    for sub in ([6, 0, 2], [9, 7], [6]):
        res = agree(eng, ora, sub)
        assert res[1] == [f for f in full[1] if f[0] in sub]
        assert res[0][:3] == (len(sub), sum(R - (g == 7) for g in sub), sum(g == 7 for g in sub))


def test_read_only_on_device_code():
    case_read_only(_emu)


def test_arguments_on_device_code():
    case_arguments(_emu)


def test_verify_structs_match_header(tmp_path):
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "josefine_raft_abi.h"\n'
                   'int main(){printf("%zu %zu %zu %zu %zu %zu %zu %d %d\\n",sizeof(jr_verify_report),sizeof(jr_verify_finding),'
                   'offsetof(jr_verify_report,leader_conflicts),offsetof(jr_verify_finding,node_mask),'
                   'offsetof(jr_verify_finding,id),offsetof(jr_verify_finding,term),offsetof(jr_verify_finding,ref_node),'
                   'JR_VERIFY_BELOW_FLOOR,JR_VERIFY_LEADER_CONFLICT);return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(abi.VerifyReport), C.sizeof(abi.VerifyFinding), abi.VerifyReport.leader_conflicts.offset,
                   abi.VerifyFinding.node_mask.offset, abi.VerifyFinding.id.offset, abi.VerifyFinding.term.offset,
                   abi.VerifyFinding.ref_node.offset, abi.VERIFY_BELOW_FLOOR, abi.VERIFY_LEADER_CONFLICT]
    assert got[:2] == [64, 32]


# ---- GPU ---------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("R", [3, 5, 7])
def test_history_on_gpu(R, monkeypatch):
    case_history(_gpu, R, monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [100, 103])
def test_random_scripts_on_gpu(seed, monkeypatch):
    case_random_script(_gpu, seed, monkeypatch, rounds=12)


@pytest.mark.gpu
def test_steady_state_is_clean_on_gpu():
    for R in range(2, 9):
        case_steady_clean(_gpu, R, G=600)


@pytest.mark.gpu
def test_constructed_violations_on_gpu():
    case_restored_chains(_gpu)
    case_forged_extend(_gpu)
    case_two_leaders_and_skips(_gpu)
    case_below_floor(_gpu)


@pytest.mark.gpu
def test_read_only_and_arguments_on_gpu():
    case_read_only(_gpu)
    case_arguments(_gpu)


def _full_size(margin, ticks):
    G, R = 65536, 5
    eng = _gpu(G, R, seed=1, chain_capacity=512)
    _bootstrap(eng, G, R)
    eng.set_auto_truncate(margin)
    eng.run(100, 100, 8, 1)
    eng.leader_table()
    now = 900
    for k in range(ticks // 64):
        eng.run_token_runs(now, 100, 64, [((k + 1) << 40 | (g + 1), 1 << 20) for g in range(G)])
        now += 6400
    assert eng.fault_count() == 0 and eng.fold_count() == G
    return eng, now


@pytest.mark.gpu
def test_full_size_clean_and_forged_65536x5():
    """65,536 x 5 after 256 ticks of jr_run_token_runs with auto-truncate 8: no findings.  Then node 2 of 1% of the
    groups restarted from an export with one token changed: exactly those groups are reported, and a subset check of
    them equals the restatement."""
    G, R = 65536, 5
    eng, now = _full_size(8, 256)
    assert _t(eng.verify_groups()) == ((G, G * R, 0, 0, 0, 0, 0, 0), [])
    forged = list(range(7, G, 100))
    exp = eng.chain_export_many([(g, 2) for g in forged])
    chains = []
    for g, (c, ck, blocks) in zip(forged, exp):
        assert len(blocks) >= 3
        chains.append((g, 2, [(i, n, t + 1 if i == c - 2 else t) for i, n, t in blocks], c, ck))
    eng.node_restart_many(now, chains)
    rep, findings = _t(eng.verify_groups())
    assert rep == (G, G * R, 0, 0, 0, 0, len(forged), 0)
    assert [(f[0], f[1], f[2], f[3], f[5]) for f in findings] == \
        [(g, abi.VERIFY_DIVERGED, 2, 1, c - 2) for g, (c, _, _) in zip(forged, exp)]
    sample = forged[::13] + [0, 1, G - 1]
    assert agree(eng, None, sample)[1] == [f for f in findings if f[0] in sample]


@pytest.mark.gpu
def test_full_size_full_windows_65536x5():
    """The same size with no truncation: 448 ticks fill most of each 512-id window, and every walk covers it."""
    G, R = 65536, 5
    eng, _ = _full_size(None, 448)
    assert int(eng.query(0, 1).commit) > 400 and int(eng.query(G - 1, 5).chain_floor) == 0
    assert _t(eng.verify_groups()) == ((G, G * R, 0, 0, 0, 0, 0, 0), [])
    sample = list(range(0, G, 4099))
    assert agree(eng, None, sample) == ((len(sample), len(sample) * R, 0, 0, 0, 0, 0, 0), [])
