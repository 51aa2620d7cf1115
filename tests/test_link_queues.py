"""Link queues (JR_F_LINK_QUEUES, deviation D8): mail sent over a cut peer link waits in a bounded per-link queue and is
delivered at the first delivery after the heal, as josefine's per-peer channel does (tcp.rs:63,90-92,110-135).  Checked
against the oracle's restatement of the queues (tests/oracle_queues) in every stepping path, with restarts, liveness
changes, truncation, steps without delivery, checkpoints and group moves; an engine with the flag and no cut computes
exactly what an engine with JR_F_PEER_LINKS only computes."""
import ctypes as C
import hashlib
import random
import struct

import numpy as np
import pytest

from josefine_b200 import abi, Command, RaftError, link_cut, partition
from josefine_b200.raft import fsm_tuple, msg_tuple
from tests.golden_scenarios import bootstrap
from tests.test_links import (Clock, ResponseRef, drain_bytes, play, random_calls, response_arrays, snapshot,
                              snapshot_group, valid_mask)

CAP, RESP, DIG, LINKS, NOFOLD, QUEUES = (abi.F_CAPTURE_FSM, abi.F_CLIENT_RESPONSES, abi.F_STREAM_DIGEST, abi.F_PEER_LINKS,
                                         abi.F_NO_SYMMETRIC_FOLD, abi.F_LINK_QUEUES)
MSGS = abi.LINK_QUEUE_MSGS


def _oracle(g, r, **kw):
    from tests.oracle_queues.queues import QueueCluster
    return QueueCluster.create(g, r, n_threads=16 if g >= 1024 else 1, **kw)


def _emu(g, r, **kw):
    from tests.emu.emu import EmuEngine
    return EmuEngine.create(g, r, **kw)


def _gpu(g, r, **kw):
    from josefine_b200 import RaftEngine
    return RaftEngine.create(g, r, **kw)


def queue_groups(api):
    """The groups with mail queued on some link."""
    return set(np.nonzero(np.asarray(api.link_queues()).any(axis=1))[0].tolist())


# ---- validation --------------------------------------------------------------------------------------------------------
def test_create_needs_peer_links():
    from tests.emu.emu import EmuEngine
    with pytest.raises(RaftError) as e:
        EmuEngine.create(8, 3, flags=QUEUES)
    assert e.value.status == abi.E_INVAL
    EmuEngine.create(8, 3, flags=QUEUES | LINKS).close()


@pytest.mark.parametrize("make", [_emu, _oracle], ids=["emu", "oracle"])
def test_refused_queries_change_nothing(make):
    G, R = 40, 3
    plain = make(G, R, seed=2, flags=LINKS)
    with pytest.raises(RaftError) as e:
        plain.link_queues()
    assert e.value.status == abi.E_INVAL
    api = make(G, R, seed=2, flags=LINKS | QUEUES)
    api.step(0, flags=0, inject=bootstrap(G, R))
    api.run(100, 100, 4)
    api.set_links([partition(R, [1])], groups=[5])
    api.run(500, 100, 3)
    before = (api.state_digest(), snapshot(api, G, R), api.link_queues().tolist())
    assert any(before[2][5])
    for groups in ([G], [1, 1], [0, G + 3]):
        with pytest.raises(RaftError) as e:
            api.link_queues(groups)
        assert e.value.status == abi.E_INVAL
    assert (api.state_digest(), snapshot(api, G, R), api.link_queues().tolist()) == before
    assert api.link_queues([5, 0]).tolist() == [before[2][5], before[2][0]]


# ---- flag on, no cut: exactly the engine without it ------------------------------------------------------------------------
@pytest.mark.parametrize("R", [3, 5, 7])
def test_no_cut_is_bit_exact_with_links_only(R):
    G = 40
    cfg = dict(seed=R + 11, chain_capacity=48, fsm_units=96)
    a, b = _emu(G, R, flags=CAP | RESP | LINKS | QUEUES, **cfg), _emu(G, R, flags=CAP | RESP | LINKS, **cfg)
    ca, cb, cap = Clock(), Clock(), G * R * 400
    folded = 0
    for i, call in enumerate(random_calls(random.Random(R + 100), G, R, 30, links=False)):
        play(a, G, R, call, ca)
        play(b, G, R, call, cb)
        assert a.state_digest() == b.state_digest() and a.fold_count() == b.fold_count(), i
        folded += a.fold_count()
        assert snapshot(a, G, R) == snapshot(b, G, R), i
        assert drain_bytes(a, cap) == drain_bytes(b, cap), i
        assert [bytes(x) for x in a.fsm_responses()[0]] == [bytes(x) for x in b.fsm_responses()[0]], i
    assert not a.link_queues().any() and folded > 0


def test_no_cut_stream_digests_equal():
    G, R = 24, 5
    cfg = dict(seed=5, chain_capacity=48, fsm_units=96, flags=CAP | DIG | LINKS)
    a, b = _emu(G, R, **{**cfg, "flags": cfg["flags"] | QUEUES}), _emu(G, R, **cfg)
    ca, cb = Clock(), Clock()
    for i, call in enumerate(random_calls(random.Random(3), G, R, 20, links=False)):
        play(a, G, R, call, ca)
        play(b, G, R, call, cb)
        assert a.stream_digest() == b.stream_digest() and a.state_digest() == b.state_digest(), i


# ---- random scripts against the oracle -----------------------------------------------------------------------------------
def queue_calls(rng, G, R, n_calls):
    """random_calls with more cuts, re-cuts before any delivery and steps that deliver nothing."""
    calls = random_calls(rng, G, R, n_calls)
    out = []
    for c in calls:
        out.append(c)
        x = rng.random()
        if x < 0.12:
            out.append(("quiet",))                   # a step without JR_STEP_DELIVER
        elif x < 0.2 and c[0] == "links":
            gs = rng.sample(range(G), rng.randint(1, G // 3))   # a re-cut before any delivery
            out.append(("links", [partition(R, rng.sample(range(1, R + 1), rng.randint(1, R // 2 + 1))) for _ in gs], gs))
        elif x < 0.3:
            out += [("links", [0] * G, None), ("run", 3, 0), ("run", 12, 1)]   # a heal, the replay, a steady run
        elif x < 0.4:   # jr_run_token_runs: per group a base (0: none) and a stride
            runs = [(0, 0) if rng.random() < 0.25 else (rng.randrange(1, 1 << 40), rng.randint(1, 1000)) for _ in range(G)]
            out.append(("token_runs", rng.randint(1, 8), runs))
    return out


def play_q(api, G, R, call, clock):
    if call[0] == "quiet":
        clock.now += 100
        return [fsm_tuple(f) for f in api.step(clock.now - 100, flags=abi.STEP_TICK).fsm]
    if call[0] == "token_runs":
        api.leader_table()
        api.run_token_runs(clock.now, 100, call[1], call[2])
        clock.now += 100 * call[1]
        return None
    return play(api, G, R, call, clock)


@pytest.mark.parametrize("R", [3, 5, 7])
@pytest.mark.parametrize("digest", [False, True], ids=["fold", "digest"])
def test_random_scripts_match_oracle(R, digest):
    G = 40
    rng = random.Random(3000 * R + digest)
    flags = CAP | LINKS | QUEUES | (DIG if digest else 0)
    # (a replay is a burst: each queued HeartbeatResponse can make a leader replicate to every peer in the same tick, so a
    #  leader of R = 7 may emit far more than mailbox_units = 128 holds; that is JR_FAULT_ENGINE_MAILBOX_OVERFLOW, an
    #  engine limit the oracle does not have)
    cfg = dict(seed=R + 40, chain_capacity=48, fsm_units=96, mailbox_units=1024)
    eng, ora = _emu(G, R, flags=flags, **cfg), _oracle(G, R, flags=flags, **cfg)
    cap, ce, co = G * R * 400, Clock(), Clock()
    folded = queued = 0
    for i, call in enumerate(queue_calls(rng, G, R, 40)):
        assert play_q(eng, G, R, call, ce) == play_q(ora, G, R, call, co), (i, call[0])
        if call[0] in ("run", "tokens", "token_runs"):
            folded += eng.fold_count()
        dq = eng.link_queues()
        assert dq.tolist() == ora.link_queues().tolist(), (i, call[0])
        queued += int(dq.sum())
        assert eng.links() == ora.links(), (i, call[0])
        assert eng.state_digest() == ora.state_digest(), (i, call[0])
        assert eng.fault_count() == ora.fault_count()
        if digest:
            assert eng.stream_digest() == ora.stream_digest(), (i, call[0])
        assert snapshot(eng, G, R) == snapshot(ora, G, R), (i, call[0])
        assert drain_bytes(eng, cap) == drain_bytes(ora, cap), (i, call[0])
    assert queued > 0
    if not digest:
        assert folded > 0


# ---- saturation ----------------------------------------------------------------------------------------------------------
def test_long_cut_keeps_the_first_messages():
    """A cut long enough to fill every link: each receiver gets exactly the first JR_LINK_QUEUE_MSGS Messages of it."""
    G, R = 16, 5
    cfg = dict(seed=8, flags=CAP | LINKS | QUEUES | abi.F_CAPTURE_MESSAGES, chain_capacity=64, fsm_units=96)
    eng, ora = _emu(G, R, **cfg), _oracle(G, R, **cfg)
    for api in (eng, ora):
        api.step(0, flags=0, inject=bootstrap(G, R))
        api.run(100, 100, 6, 1)
    full = partition(R, [1, 2])
    sent = {}   # (g, s, r) -> the Messages s emitted for r that were delivered while the link was cut, in order
    now = 700
    for t in range(15):
        if t == 1:   # the mail of step 0 is the first the cut meets
            for api in (eng, ora):
                api.set_links([full] * G)
        res = [api.step(now, flags=abi.STEP_DELIVER | abi.STEP_TICK | abi.STEP_SYNTH_PROPOSALS, n_synth=1) for api in (eng, ora)]
        assert [msg_tuple(m) for m in res[0].messages] == [msg_tuple(m) for m in res[1].messages], t
        if t < 14:   # (the last step's mail is delivered after the heal, not queued)
            for m in res[0].messages:
                for r in range(1, R + 1):
                    if m.from_id != r and (full >> (8 * (r - 1) + (m.from_id - 1))) & 1 and \
                            (m.to_kind == abi.ADDR_PEERS or (m.to_kind == abi.ADDR_PEER and m.to_id == r)):
                        sent.setdefault((m.group, m.from_id, r), []).append(msg_tuple(m))
        now += 100
        assert eng.link_queues().tolist() == ora.link_queues().tolist(), t
    dq = eng.link_queues()
    for g in range(G):
        for s in range(1, R + 1):
            for r in range(1, R + 1):
                if (full >> (8 * (r - 1) + (s - 1))) & 1:
                    assert dq[g, 8 * (r - 1) + (s - 1)] == min(MSGS, len(sent.get((g, s, r), []))), (g, s, r)
    assert (dq == MSGS).sum() > 0
    # after the heal the first delivery replays the queues, and they are empty
    for api in (eng, ora):
        api.set_links([0] * G)
    res = [api.step(now) for api in (eng, ora)]
    assert [msg_tuple(m) for m in res[0].messages] == [msg_tuple(m) for m in res[1].messages]
    assert not eng.link_queues().any() and not ora.link_queues().any()
    assert snapshot(eng, G, R) == snapshot(ora, G, R) and eng.state_digest() == ora.state_digest()


def test_vote_request_copies_fit_partly():
    """An isolated R = 5 follower keeps seeking election: each VoteRequest is 4 copies, and the copies that do not fit in
    the queue are dropped one by one."""
    G, R = 8, 5
    cfg = dict(seed=12, flags=CAP | LINKS | QUEUES, chain_capacity=64, fsm_units=96)
    eng, ora = _emu(G, R, **cfg), _oracle(G, R, **cfg)
    for api in (eng, ora):
        api.step(0, flags=0, inject=bootstrap(G, R))
        api.run(100, 100, 6, 1)
        api.node_restart_many(700, [(g, 5, None, 0, None) for g in range(G)])   # voted_for = 0: it may seek election
        api.set_links([partition(R, [5])] * G)
        # a VoteRequest from node 2 (injected: the host is its network): node 5's VoteResponse is the first Message on
        # link 5 -> 2, so the VoteRequests that follow do not fill it in whole copies
        api.step(700, inject=[Command.vote_request(g, 5, 1, 2, 1, 0) for g in range(G)])
    seen = set()
    for t in range(1, 60):
        for api in (eng, ora):
            api.run(700 + 100 * t, 100, 1, 1)
        dq, do = eng.link_queues(), ora.link_queues()
        assert dq.tolist() == do.tolist(), t
        assert eng.state_digest() == ora.state_digest(), t
        seen |= set(dq[:, 8 * 1 + 4].tolist())    # link 5 -> 2
    assert MSGS in seen and any(v % (R - 1) for v in seen if v)   # full, and reached through a partial VoteRequest
    assert max(st.current_term for st in eng.query_many([(g, 5) for g in range(G)])) >= 3


# ---- stale mail after a partition ---------------------------------------------------------------------------------------
def stale_mail(make, queues):
    """R = 3: the leader is cut off, both followers restart and elect a new leader in a new term, then the cut heals."""
    G, R = 4, 3
    flags = CAP | LINKS | (QUEUES if queues else 0)
    cfg = dict(seed=17, flags=flags, chain_capacity=64, fsm_units=96)
    eng, ora = make(G, R, **cfg), _oracle(G, R, **cfg)
    now = 100
    for api in (eng, ora):
        api.step(0, flags=0, inject=bootstrap(G, R))
        api.run(now, 100, 6, 1)
    now += 600
    leaders = [l for _t, l, _c in eng.leader_table()]
    assert all(leaders)
    for api in (eng, ora):
        api.set_links([partition(R, [l]) for l in leaders])
    trace = []

    def tick(k=1):
        nonlocal now
        for _ in range(k):
            for api in (eng, ora):
                api.run(now, 100, 1, 1)
            now += 100
            assert eng.state_digest() == ora.state_digest(), now
            if queues:
                assert eng.link_queues().tolist() == ora.link_queues().tolist(), now
            trace.append([(s.role, s.fault, s.current_term) for s in eng.query_many([(g, n) for g in range(G) for n in (1, 2, 3)])])

    tick(3)
    for api in (eng, ora):
        api.node_restart_many(now, [(g, n, None, 0, None) for g in range(G) for n in range(1, R + 1) if n != leaders[g]])
    tick(25)   # the followers' timers run out: a new leader in a new term
    new = [[n for n in range(1, R + 1) if eng.query(g, n).role == abi.ROLE_LEADER and n != leaders[g]] for g in range(G)]
    for api in (eng, ora):
        api.set_links([0] * G)
    tick(4)
    assert snapshot(eng, G, R) == snapshot(ora, G, R)
    faults = {(g, n): eng.query(g, n).fault for g in range(G) for n in range(1, R + 1)}
    return leaders, new, faults


def _stale(make):
    """The engine equals the oracle tick for tick, with queues and without (stale_mail).  What the oracle shows is not the
    pair of faults one might expect from follower.rs:146-153 and leader.rs:33-35 (DESIGN.md section 3g, "Stale mail"): a
    restarted node starts again at term 0 (State is not persisted), so the new leader's term does not exceed the old
    leader's and the old leader never sees a later term; the new leader, reopened in place with head above commit, faults
    on its first append (IdGenerator::new(commit), chain.rs:126,160-175); and the old leader's fresh AppendEntries after
    the heal carry its old term as well as the queued ones, so a follower of a later term faults on them with drop
    semantics too."""
    out = [stale_mail(make, q) for q in (True, False)]
    for leaders, new, faults in out:
        G, R = len(leaders), 3
        assert all(new), new
        for g in range(G):
            assert faults[(g, leaders[g])] == abi.FAULT_NONE, (g, faults)
            assert faults[(g, new[g][0])] == abi.FAULT_APPEND_ID_NOT_GT_HEAD, (g, faults)
    assert out[0][2] == out[1][2]


def test_stale_mail_after_heal_emu():
    _stale(_emu)


# ---- carriage ------------------------------------------------------------------------------------------------------------
def _queued(make, G=40, R=5, **kw):
    cfg = dict(seed=4, flags=CAP | LINKS | QUEUES, chain_capacity=64, fsm_units=96)
    cfg.update(kw)
    api = make(G, R, **cfg)
    api.step(0, flags=0, inject=bootstrap(G, R))
    api.run(100, 100, 8, 0)
    api.set_links([partition(R, [1]), partition(R, [1, 2]), link_cut(R, [(3, 1), (2, R)])], groups=[2, 5, 9])
    api.leader_table()
    api.run_tokens(900, 100, [[(t << 20) + g + 1 for g in range(G)] for t in range(5)])
    return api


def heal_and_run(api, G):
    api.set_links([0] * G)
    api.run(1400, 100, 3, 0)
    api.leader_table()
    api.run_tokens(1700, 100, [[(9 << 20) + (t << 12) + g + 1 for g in range(G)] for t in range(8)])


def _checkpoint(make):
    G, R = 40, 5
    twin, a = _queued(make), _queued(make)
    assert a.link_queues()[[2, 5, 9]].any(axis=1).all()
    b = make(G, R, seed=4, flags=CAP | LINKS | QUEUES, chain_capacity=64, fsm_units=96)
    b.restore(a.save())
    assert b.link_queues().tolist() == a.link_queues().tolist() and b.links() == a.links()
    for api in (twin, b):
        heal_and_run(api, G)
    assert snapshot(b, G, R) == snapshot(twin, G, R) and b.state_digest() == twin.state_digest()
    assert not b.link_queues().any()


def _move(make):
    G, R = 40, 5
    twin, src = _queued(make), _queued(make)
    other = make(G, R, seed=4, group_offset=3, flags=CAP | LINKS | QUEUES, chain_capacity=64, fsm_units=96)
    cap = G * R * 400
    drain_bytes(twin, cap)
    drain_bytes(src, cap)
    before = src.link_queues([5]).tolist()
    img = src.export_groups([5])
    assert src.link_queues([5]).tolist() == before and any(before[0])   # the source slot keeps its queues
    other.import_groups([2], img)      # another engine: global id 5 again
    assert other.link_queues([2]).tolist() == before and other.links([2]) == twin.links([5])
    for api in (twin, other):
        api.set_links([0], groups=[5 if api is twin else 2])
        api.run(1400, 100, 10, 0)
    assert snapshot_group(other, 2, R) == snapshot_group(twin, 5, R)
    assert not other.link_queues([2]).any()
    # within one engine, to another slot (whose global id, and so its election timeouts, differ): the slot gets the
    # image's queues, the source keeps its own, and the first delivery after the heal empties both
    same = _queued(make)
    drain_bytes(same, cap)
    q9 = same.link_queues([9]).tolist()
    same.import_groups([30], same.export_groups([9]))
    assert same.link_queues([30, 9]).tolist() == q9 * 2 and same.links([30]) == same.links([9])
    same.set_links([0] * G)
    same.run(1400, 100, 1, 0)
    assert not same.link_queues().any()


def _reset(make):
    G, R = 40, 5
    api = _queued(make)
    assert api.link_queues().any()
    api._check(api._lib.jr_engine_reset(api._h), "engine_reset")
    assert not api.link_queues().any() and api.links() == [0] * G
    fresh = make(G, R, seed=4, flags=CAP | LINKS | QUEUES, chain_capacity=64, fsm_units=96)
    for x in (api, fresh):
        x.step(0, flags=0, inject=bootstrap(G, R))
        x.run(100, 100, 8, 0)
    assert snapshot(api, G, R) == snapshot(fresh, G, R) and api.fold_count() == fresh.fold_count()


def test_checkpoint_carries_queues_emu():
    _checkpoint(_emu)


def test_group_move_carries_queues_emu():
    _move(_emu)


def test_reset_empties_queues_emu():
    _reset(_emu)


def test_restart_drops_the_senders_queues_only():
    G, R = 12, 3
    eng, ora = _queued(_emu, G, R), _queued(_oracle, G, R)
    assert eng.link_queues().tolist() == ora.link_queues().tolist()
    before = eng.link_queues()
    for api in (eng, ora):
        api.node_restart_many(1500, [(2, 1, None, 0, None), (5, 2, None, 0, None), (5, 3, None, 0, None)])
    after = eng.link_queues()
    assert after.tolist() == ora.link_queues().tolist()
    for g, n in ((2, 1), (5, 2), (5, 3)):
        for r in range(1, R + 1):
            assert after[g, 8 * (r - 1) + (n - 1)] == 0          # from the restarted node: gone
    keep = before.copy()
    for g, n in ((2, 1), (5, 2), (5, 3)):
        keep[g, [8 * (r - 1) + (n - 1) for r in range(1, R + 1)]] = 0
    assert (after == keep).all()                                   # everything else, queues to it included, stays
    for api in (eng, ora):
        heal_and_run(api, G)
    assert snapshot(eng, G, R) == snapshot(ora, G, R)


# A checkpoint's queues are checked on the host: a depth above the bound, units beyond a link's storage, a mask that does
# not match the depths.
def test_restore_refuses_bad_queues():
    G, R = 40, 5
    a = _queued(_emu)
    blob = bytearray(a.save())
    Gp, plane, slots = 64, 5 * 64, R - 1
    o_lq = len(blob) - plane * slots * MSGS * (1 + 5) * 16
    o_lqc = o_lq - plane * slots * 4
    o_lqm = o_lqc - Gp * 8
    b = _emu(G, R, seed=4, flags=CAP | LINKS | QUEUES, chain_capacity=64, fsm_units=96)
    b.restore(bytes(blob))          # (the offsets are right: the unmodified blob is accepted)
    before = (b.state_digest(), b.link_queues().tolist())
    g = 5
    mask = struct.unpack_from("<Q", blob, o_lqm + 8 * g)[0]
    bit = (mask & -mask).bit_length() - 1
    r, s = bit // 8, bit % 8
    at = o_lqc + 4 * ((s - (s > r)) * plane + r * Gp + g)
    c = struct.unpack_from("<I", blob, at)[0]
    for bad_c, bad_mask in ((MSGS + 1 | (c & ~255), mask), ((c & 255) | (49 << 8), mask), (c, mask & ~(1 << bit)),
                            (0, mask), (c, mask | (1 << 63))):
        x = bytearray(blob)
        struct.pack_into("<I", x, at, bad_c)
        struct.pack_into("<Q", x, o_lqm + 8 * g, bad_mask)
        with pytest.raises(RaftError) as e:
            b.restore(bytes(x))
        assert e.value.status == abi.E_INVAL
    assert (b.state_digest(), b.link_queues().tolist()) == before


# Engines with JR_F_PEER_LINKS only keep their checkpoint size and their group images, byte for byte (record padding
# and the checksum over it aside: those bytes were never written); the values were taken from the engine before link
# queues existed (host build), mid-cut, with this script.
LINKS_ONLY = {
    3: (1220616, 3200, "4a8a77e6eef414dc623c40dc29d2b99846fe5eb1584673b42d874a5f8fb8376f"),
    5: (2038792, 5024, "28dedd28a012fcfedc2caf9a4c4da3f13adc45a1a4cd4f2b581fdbfd5edeac88"),
}


def image_without_padding(img, R, n):
    hs = 8 + 4 + 4 + 8 + 8 + C.sizeof(abi.Config) + 4 + 4 + 16
    rec_units, words = struct.unpack_from("<II", img, hs - 24)
    b = bytearray(img)
    b[24:32] = bytes(8)
    for t in range(R * n):
        at = hs + 16 * (t * rec_units + 1)
        b[at + 4 * words: at + 16 * (rec_units - 1)] = bytes(16 * (rec_units - 1) - 4 * words)
    return bytes(b)


def _links_only_layout(make):
    for R, (save_bytes, image_bytes, sha) in LINKS_ONLY.items():
        G = 40
        a = make(G, R, seed=1, flags=CAP | RESP | LINKS, chain_capacity=48, fsm_units=96)
        a.step(0, flags=0, inject=bootstrap(G, R))
        a.run(100, 100, 7, 1)
        a.set_links([partition(R, [1])] * 3, groups=[1, 7, 9])
        a.run(800, 100, 5, 1)
        img = a.export_groups([1, 7])
        assert (len(a.save()), len(img), hashlib.sha256(image_without_padding(img, R, 2)).hexdigest()) == \
            (save_bytes, image_bytes, sha)


def test_links_only_checkpoints_and_images_keep_their_bytes_emu():
    _links_only_layout(_emu)


# ---- the two restatements, differenced with queues --------------------------------------------------------------------------
@pytest.mark.parametrize("R", [3, 5])
def test_python_restatement_agrees_with_queues(R):
    from tests.oracle_queues.queues import PyQueueCluster
    G = 6
    cfg = dict(seed=50 + R, chain_capacity=64, flags=abi.F_CAPTURE_MESSAGES | CAP | LINKS | QUEUES)
    a, b = _oracle(G, R, **cfg), PyQueueCluster.create(G, R, **cfg)
    rng = random.Random(R + 7)
    for api in (a, b):
        api.step(0, flags=0, inject=bootstrap(G, R))
    total = 0
    for t in range(1, 150):
        if t % 12 == 0:
            gs = rng.sample(range(G), 3)
            cuts = [rng.choice([0, 0, partition(R, rng.sample(range(1, R + 1), R // 2)),
                                rng.getrandbits(64) & valid_mask(R) & rng.getrandbits(64)]) for _ in gs]
            for api in (a, b):
                api.set_links(cuts, groups=gs)
        inj = [Command.client_request(g, rng.randint(1, R), t * 100 + g) for g in range(G) if rng.random() < 0.3]
        if t % 17 == 0:
            inj.append(Command.timeout(rng.randrange(G), rng.randint(1, R)))
        flags = abi.STEP_TICK if t % 9 == 0 else abi.STEP_DELIVER | abi.STEP_TICK
        ra, rb = a.step(100 * t, flags=flags, inject=inj), b.step(100 * t, flags=flags, inject=inj)
        assert [msg_tuple(m) for m in ra.messages] == [msg_tuple(m) for m in rb.messages], t
        assert [fsm_tuple(f) for f in ra.fsm] == [fsm_tuple(f) for f in rb.fsm], t
        qa = a.link_queues().tolist()
        assert qa == b.link_queues(), t
        total += sum(map(sum, qa))
        for g in range(G):
            for n in range(1, R + 1):
                sa, sb = a.query(g, n), b.query(g, n)
                assert (sa.current_term, sa.role, sa.head, sa.commit, sa.fault, sa.leader_id, sa.voted_for) == \
                       (sb.current_term, sb.role, sb.head, sb.commit, sb.fault, sb.leader_id, sb.voted_for), (t, g, n)
    assert total > 0


# ---- fleet scale ---------------------------------------------------------------------------------------------------------
def fleet_scenario(make, G, R, quantum=64, n_before=1, n_during=3, n_after=2, check_snapshots=True):
    """Steady state with auto-truncate and tokens; isolate 10% of the leaders and partition {1,2} | {3..5} in another 5%
    of the groups; run; heal; run on.  Engine against the oracle after every quantum: state, records, ClientResponses
    and queue depths.  Returns (G, cut groups, fold counts during the cut, groups with queued mail at the heal, fold
    count of the launch after the heal)."""
    cfg = dict(seed=23, chain_capacity=128, fsm_units=64)
    eng = make(G, R, flags=CAP | RESP | LINKS | QUEUES, **cfg)
    ora = _oracle(G, R, flags=CAP | LINKS | QUEUES, **cfg)
    apis = (eng, ora)
    cap = G * R * 2 * quantum + 4096   # (Instructions per replica and tick: at most two in steady state)
    now = 100
    for api in apis:
        api.step(0, flags=0, inject=bootstrap(G, R))
        api.set_auto_truncate(6)
        api.run(now, 100, 24, 1)
    now += 2400
    ref = ResponseRef()

    def compare(k):
        want = drain_bytes(ora, cap)
        assert drain_bytes(eng, cap) == want, k
        runs, batch = eng.fsm_responses()
        got, exp = response_arrays(runs), ref.feed(want)
        assert batch.n_dropped == 0 and len(got) == len(exp) and (got == exp).all(), k
        assert eng.state_digest() == ora.state_digest(), k
        assert eng.leader_table() == ora.leader_table(), k
        assert (eng.link_queues() == ora.link_queues()).all(), k
        if check_snapshots:
            assert snapshot(eng, G, R) == snapshot(ora, G, R), k

    compare("bootstrap")
    step = [0]

    def quantum_step():
        nonlocal now
        k = step[0]
        step[0] += 1
        toks = [[((k * quantum + t) << 24 | g) + 1 for g in range(G)] for t in range(quantum)]
        for api in apis:
            api.leader_table()
            api.run_tokens(now, 100, toks)
        now += 100 * quantum
        compare(k)
        return eng.fold_count()

    for _ in range(n_before):
        assert quantum_step() == G
    n = [api.isolate_leaders(5, 100) for api in apis]
    assert n[0] == n[1] > 0
    iso = {g for g, m in enumerate(eng.links()) if m}
    part = [g for g in range(G) if g % 20 == 3 and g not in iso]
    for api in apis:
        api.set_links([partition(R, [1, 2])] * len(part), groups=part)
    cut = sum(1 for m in eng.links() if m)
    during = [quantum_step() for _ in range(n_during)]
    queued = queue_groups(eng)
    for api in apis:
        api.set_links([0] * G)
    after = [quantum_step() for _ in range(n_after)]
    assert not eng.link_queues().any()
    return cut, during, queued, after


def test_fleet_scenario_emu():
    G, R = 256, 5
    cut, during, queued, after = fleet_scenario(_emu, G, R, quantum=16)
    assert during == [G - cut] * len(during)
    assert queued and after[0] <= G - len(queued)


@pytest.mark.gpu
def test_fleet_scenario_gpu_65536():
    G, R = 65536, 5
    cut, during, queued, after = fleet_scenario(_gpu, G, R, check_snapshots=False)
    assert cut > G // 10
    assert during == [G - cut] * len(during)          # every group without a cut folds, no group with one does
    assert len(queued) > G // 10 and after[0] <= G - len(queued)   # no group with queued mail folds after the heal


@pytest.mark.gpu
def test_no_cut_is_bit_exact_gpu_65536():
    G, R = 65536, 5
    cfg = dict(seed=31, chain_capacity=128, fsm_units=64)
    a, b = _gpu(G, R, flags=CAP | RESP | LINKS | QUEUES, **cfg), _gpu(G, R, flags=CAP | RESP | LINKS, **cfg)
    cap = G * R * 4 * 64 + 4096
    for api in (a, b):
        api.step(0, flags=0, inject=bootstrap(G, R))
        api.set_auto_truncate(6)
    now = 100
    for k in range(4):
        toks = [[((k * 64 + t) << 24 | g) + 1 for g in range(G)] for t in range(64)]
        for api in (a, b):
            api.leader_table()
            api.run_tokens(now, 100, toks) if k else api.run(now, 100, 24, 1)
        now += 6400
        assert a.state_digest() == b.state_digest() and a.fold_count() == b.fold_count(), k
        assert drain_bytes(a, cap) == drain_bytes(b, cap), k
        assert [bytes(x) for x in a.fsm_responses()[0]] == [bytes(x) for x in b.fsm_responses()[0]], k
    assert a.fold_count() == G and not a.link_queues().any()


@pytest.mark.gpu
def test_random_scripts_gpu():
    for R in (3, 5, 7):
        G = 40
        rng = random.Random(11 * R)
        flags = CAP | LINKS | QUEUES
        cfg = dict(seed=R, chain_capacity=48, fsm_units=96, mailbox_units=1024)   # (see test_random_scripts_match_oracle)
        eng, ora = _gpu(G, R, flags=flags, **cfg), _oracle(G, R, flags=flags, **cfg)
        ce, co, cap = Clock(), Clock(), G * R * 400
        for i, call in enumerate(queue_calls(rng, G, R, 36)):
            assert play_q(eng, G, R, call, ce) == play_q(ora, G, R, call, co), (R, i)
            assert eng.link_queues().tolist() == ora.link_queues().tolist(), (R, i)
            assert eng.state_digest() == ora.state_digest(), (R, i)
            assert snapshot(eng, G, R) == snapshot(ora, G, R), (R, i)
            assert drain_bytes(eng, cap) == drain_bytes(ora, cap), (R, i)


@pytest.mark.gpu
def test_stale_mail_after_heal_gpu():
    _stale(_gpu)


@pytest.mark.gpu
def test_carriage_gpu():
    _checkpoint(_gpu)
    _move(_gpu)
    _reset(_gpu)
    _links_only_layout(_gpu)
