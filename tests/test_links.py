"""Peer-link cuts (JR_F_PEER_LINKS: jr_set_links / jr_get_links / jr_isolate_leaders, deviation D8): directional cuts and
partitions between a group's replicas, leader isolation and heal, checked against the oracle's restatement of the same
calls (tests/oracle_links) in every stepping path -- jr_step with injected mail, jr_run, jr_run_tokens, the fold's
launches -- together with restarts, liveness changes, truncation, checkpoints and group moves.  An engine with the flag
and every matrix at zero computes exactly what an engine without it computes."""
import ctypes as C
import random

import numpy as np
import pytest

from josefine_b200 import abi, Command, RaftError, link_cut, partition
from josefine_b200.raft import expand_responses, fsm_tuple
from tests.golden_scenarios import bootstrap

CAP, RESP, DIG, LINKS, NOFOLD = (abi.F_CAPTURE_FSM, abi.F_CLIENT_RESPONSES, abi.F_STREAM_DIGEST, abi.F_PEER_LINKS,
                                 abi.F_NO_SYMMETRIC_FOLD)


def _oracle(g, r, **kw):
    from tests.oracle_links.links import LinkCluster
    return LinkCluster.create(g, r, n_threads=16 if g >= 1024 else 1, **kw)


def _emu(g, r, **kw):
    from tests.emu.emu import EmuEngine
    return EmuEngine.create(g, r, **kw)


def _gpu(g, r, **kw):
    from josefine_b200 import RaftEngine
    return RaftEngine.create(g, r, **kw)


def snapshot(api, G, R):
    tg = [(g, n) for g in range(G) for n in range(1, R + 1)]
    st = [(s.current_term, s.voted_for, s.leader_id, s.election_time_ms, s.election_timeout_ms, s.rng_draws, s.head,
           s.commit, s.id_gen, s.max_key, s.heartbeat_time_ms, s.votes_seen, s.votes_granted, tuple(s.progress_head),
           s.progress_replicate, s.role, s.fault, s.alive, s.n_queued, s.chain_floor) for s in api.query_many(tg)]
    return st, api.chain_read_many([(g, n, s[19], 24) for (g, n), s in zip(tg, st)])


def drain_bytes(api, cap):
    """Every undrained Instruction, as the raw bytes of jr_drain_fsm's array (cheap to compare at any size)."""
    buf, n = (abi.FsmInstr * cap)(), C.c_size_t(0)
    api._check(api._fn("drain_fsm")(api._h, buf, C.c_size_t(cap), C.byref(n)), "drain_fsm")
    return C.string_at(buf, n.value * C.sizeof(abi.FsmInstr))


def valid_mask(R):
    return link_cut(R, [(s, r) for s in range(1, R + 1) for r in range(1, R + 1) if s != r]) if R > 1 else 0


# ---- pure helpers ------------------------------------------------------------------------------------------------------
def test_link_cut_and_partition_bits():
    assert link_cut(3, [(1, 2)]) == 1 << 8            # receiver 2's row, sender 1's bit
    assert link_cut(3, [(3, 1)]) == 1 << 2
    assert partition(5, [1, 2]) == partition(5, [3, 4, 5])
    p = partition(3, [1])
    assert p == link_cut(3, [(1, 2), (1, 3), (2, 1), (3, 1)])
    assert partition(5, []) == 0 and partition(5, range(1, 6)) == 0
    with pytest.raises(ValueError):
        link_cut(3, [(2, 2)])
    with pytest.raises(ValueError):
        link_cut(3, [(1, 4)])


# ---- validation --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("make", [_emu, _oracle], ids=["emu", "oracle"])
def test_refused_calls_change_nothing(make):
    G, R = 40, 3
    plain = make(G, R, seed=2)
    for call in (lambda: plain.set_links([0] * G), lambda: plain.links(), lambda: plain.isolate_leaders(1, 1000)):
        with pytest.raises(RaftError) as e:
            call()
        assert e.value.status == abi.E_INVAL
    api = make(G, R, seed=2, flags=LINKS)
    api.step(0, flags=0, inject=bootstrap(G, R))
    api.run(100, 100, 4)
    api.set_links([partition(R, [2]), link_cut(R, [(1, 3)])], groups=[5, 39])
    want = [0] * G
    want[5], want[39] = partition(R, [2]), link_cut(R, [(1, 3)])
    assert api.links() == want and api.links([39, 5]) == [want[39], want[5]]
    before = (api.state_digest(), snapshot(api, G, R))
    bad = [
        ([1 << 0], [3]),                          # diagonal: 1 -> 1
        ([1 << (8 * 1 + 1)], [3]),                # diagonal: 2 -> 2
        ([1 << 3], [3]),                          # sender 4 of 3
        ([1 << (8 * 3)], [3]),                    # receiver 4 of 3
        ([1 << 63], [3]),
        ([0, 1 << 8], [3, 3]),                    # a group named twice
        ([1 << 8], [G]),                          # out of range
        ([1 << 8, 1 << 9], [0, G + 7]),
    ]
    for cuts, groups in bad:
        with pytest.raises(RaftError) as e:
            api.set_links(cuts, groups=groups)
        assert e.value.status == abi.E_INVAL, (cuts, groups)
    for cuts in ([0] * (G - 1), [0] * (G + 1)):   # dense form: exactly one matrix per group
        with pytest.raises(RaftError):
            api.set_links(cuts)
    for groups in ([G], [1, 1]):
        with pytest.raises(RaftError):
            api.links(groups)
    assert api.links() == want
    assert (api.state_digest(), snapshot(api, G, R)) == before
    api.set_links([0] * G)
    assert api.links() == [0] * G


# ---- random scripts against the oracle -----------------------------------------------------------------------------------
class DriverRef:
    """fsm::Driver's notification map over the oracle's Instructions (fsm.rs:57-81)."""

    def __init__(self):
        self.maps = {}

    def feed(self, instructions):
        out = []
        for g, n, kind, ckind, cid, bid, _nxt, data in instructions:   # fsm_tuple form
            m = self.maps.setdefault((g, n), {})
            if kind == abi.FSM_NOTIFY:
                m[bid] = (ckind, cid, data)
            elif bid != 0 and bid in m:
                out.append((g, n) + m.pop(bid) + (bid,))
        return sorted(out, key=lambda x: (x[0], x[1]))


def random_calls(rng, G, R, n_calls, links=True):
    """A seeded script: (name, args) tuples.  links=False: the same kind of script without a single link call."""
    kinds = ["run", "run", "tokens", "tokens", "step", "alive", "trunc", "restart"]
    if links:
        kinds += ["cut", "cut", "partition", "heal", "isolate"]
    calls = [("boot",)]
    for _ in range(n_calls):
        k = rng.choice(kinds)
        if k == "run":
            calls.append(("run", rng.randint(1, 12), rng.choice([0, 1, 2])))
        elif k == "tokens":
            n = rng.randint(1, 8)
            base = rng.randrange(1, 1 << 40)
            quiet = set(rng.sample(range(G), G // 4))     # (per group one arithmetic run: the notification map holds it)
            calls.append(("tokens", [[0 if g in quiet else base + 1000 * t + g for g in range(G)] for t in range(n)]))
        elif k == "step":
            inj = [Command.client_request(g, rng.randint(1, R), rng.randrange(1, 1 << 40)) for g in rng.sample(range(G), G // 4)]
            inj += [Command.timeout(g, rng.randint(1, R)) for g in rng.sample(range(G), 2)]
            calls.append(("step", inj))
        elif k == "alive":
            calls.append(("alive", [(rng.randrange(G), rng.randint(1, R), rng.random() < 0.6) for _ in range(3)]))
        elif k == "trunc":
            calls.append(("trunc", rng.choice([None, 2, 6, "now"])))
        elif k == "restart":
            calls.append(("restart", [(g, rng.randint(1, R), None, 0, None) for g in rng.sample(range(G), 3)]))
        elif k == "cut":
            gs = rng.sample(range(G), rng.randint(1, G // 3))
            calls.append(("links", [rng.getrandbits(64) & valid_mask(R) & rng.getrandbits(64) for _ in gs], gs))
        elif k == "partition":
            gs = rng.sample(range(G), rng.randint(1, G // 2))
            calls.append(("links", [partition(R, rng.sample(range(1, R + 1), rng.randint(1, R // 2 + 1))) for _ in gs], gs))
        elif k == "heal":
            calls.append(("links", [0] * G, None))
        else:
            calls.append(("isolate", rng.randrange(1 << 32), rng.choice([200, 500, 1000])))
    return calls


class Clock:
    def __init__(self):
        self.now = 100


def play(api, G, R, call, clock):
    name = call[0]
    if name == "boot":
        api.step(0, flags=0, inject=bootstrap(G, R))
        api.run(clock.now, 100, 6, 1)
        clock.now += 600
    elif name == "run":
        api.run(clock.now, 100, call[1], call[2])
        clock.now += 100 * call[1]
    elif name == "tokens":
        api.leader_table()
        api.run_tokens(clock.now, 100, call[1])
        clock.now += 100 * len(call[1])
    elif name == "step":
        clock.now += 100
        return [fsm_tuple(f) for f in api.step(clock.now - 100, inject=call[1]).fsm]   # the step takes its Instructions
    elif name == "alive":
        for g, n, a in call[1]:
            api.set_alive(g, n, a)
    elif name == "trunc":
        if call[1] == "now":
            api.truncate(4)
        else:
            api.set_auto_truncate(call[1])
    elif name == "restart":
        api.node_restart_many(clock.now, call[1])
    elif name == "links":
        api.set_links(call[1], groups=call[2])
    elif name == "isolate":
        return api.isolate_leaders(call[1], call[2])


@pytest.mark.parametrize("R", [3, 5, 7])
@pytest.mark.parametrize("digest", [False, True], ids=["fold", "digest"])
def test_random_scripts_match_oracle(R, digest):
    G = 40
    rng = random.Random(1000 * R + digest)
    flags = CAP | LINKS | (DIG if digest else 0)
    cfg = dict(seed=R, chain_capacity=48, fsm_units=96, mailbox_units=128)   # (lagging followers of R = 7: many AppendEntries runs)
    eng, ora = _emu(G, R, flags=flags | RESP, **cfg), _oracle(G, R, flags=flags, **cfg)
    ref, cap, clock_e, clock_o = DriverRef(), G * R * 400, Clock(), Clock()
    folded, exact = 0, True
    expand = lambda runs: [(g, n, to.kind, to.id, tok, bid) for g, n, to, tok, bid in expand_responses(runs)]   # noqa: E731
    for i, call in enumerate(random_calls(rng, G, R, 36)):
        res = play(eng, G, R, call, clock_e)
        assert res == play(ora, G, R, call, clock_o), (i, call[0])
        if call[0] == "step":
            runs, batch = eng.fsm_responses()
            want = ref.feed(res)
            exact = exact and batch.n_dropped == 0
            assert not exact or expand(runs) == want, (i, call[0])
        if call[0] in ("run", "tokens"):
            folded += eng.fold_count()
        assert eng.links() == ora.links(), (i, call[0])
        assert eng.state_digest() == ora.state_digest(), (i, call[0])
        assert eng.fault_count() == ora.fault_count()
        if digest:
            assert eng.stream_digest() == ora.stream_digest(), (i, call[0])
        assert snapshot(eng, G, R) == snapshot(ora, G, R), (i, call[0])
        ins = [fsm_tuple(f) for f in ora.drain_fsm(cap=cap)]
        assert [fsm_tuple(f) for f in eng.drain_fsm(cap=cap)] == ins, (i, call[0])
        runs, batch = eng.fsm_responses()
        if call[0] == "restart":   # a new process gets a new Driver (server.rs:80-81); nothing was left undrained
            for g, n, *_ in call[1]:
                ref.maps.pop((g, n), None)
        want = ref.feed(ins)
        # An isolated leader keeps taking requests it never commits: once its notification map overflows (JR_NOTIFY_RUNS,
        # counted in n_dropped) the engine's answers leave the unbounded reference map's.  The records stay exact.
        exact = exact and batch.n_dropped == 0
        assert not exact or expand(runs) == want, (i, call[0])
    if not digest:
        assert folded > 0      # the script went through the fold too


@pytest.mark.parametrize("R", [3, 5, 7])
def test_flag_with_zero_matrix_is_bit_exact(R):
    G = 40
    cfg = dict(seed=R + 1, chain_capacity=48, fsm_units=96)
    a, b = _emu(G, R, flags=CAP | RESP | LINKS, **cfg), _emu(G, R, flags=CAP | RESP, **cfg)
    ca, cb, cap = Clock(), Clock(), G * R * 400
    for i, call in enumerate(random_calls(random.Random(R), G, R, 30, links=False)):
        play(a, G, R, call, ca)
        play(b, G, R, call, cb)
        assert a.state_digest() == b.state_digest() and a.fold_count() == b.fold_count(), i
        assert snapshot(a, G, R) == snapshot(b, G, R), i
        assert drain_bytes(a, cap) == drain_bytes(b, cap), i
        assert [bytes(x) for x in a.fsm_responses()[0]] == [bytes(x) for x in b.fsm_responses()[0]], i
    assert a.links() == [0] * G


@pytest.mark.parametrize("make", [_emu, _oracle], ids=["emu", "oracle"])
def test_isolate_picks_kill_leaders_groups(make):
    G, R = 200, 5
    a, b = make(G, R, seed=9, flags=LINKS), make(G, R, seed=9, flags=LINKS)
    for api in (a, b):
        api.step(0, flags=0, inject=bootstrap(G, R))
        api.run(100, 100, 6, 1)
        api.set_alive(7, 1, False)        # a group without a live leader is picked but counts for nothing
    n_iso = a.isolate_leaders(77, 300)
    n_kill = b.kill_leaders(77, 300)
    assert n_iso == n_kill > 0
    iso = {g for g, m in enumerate(a.links()) if m}
    dead = {g for g in range(G) if not b.query(g, 1).alive and g != 7}
    assert iso == dead
    for g in iso:
        assert a.links([g]) == [partition(R, [1])]     # the leader (node 1) cut off both ways
        assert a.query(g, 1).alive
    assert a.isolate_leaders(77, 300) == n_iso          # ORed in: the same matrices again
    assert {g for g, m in enumerate(a.links()) if m} == iso


FSM_DT = np.dtype([("group", "<u4"), ("node", "<u4"), ("kind", "u1"), ("ckind", "u1"), ("res", "<u2"), ("cid", "<u4"),
                   ("id", "<u8"), ("next", "<u8"), ("data", "<u8")])
RESP_DT = np.dtype([("group", "<u4"), ("node", "<u4"), ("ckind", "<u4"), ("cid", "<u4"), ("tok", "<u8"), ("id", "<u8")])


class ResponseRef:
    """fsm::Driver's notification map (fsm.rs:57-81) over drained Instructions (jr_drain_fsm's bytes), for any size:
    Notify{id} inserts or overwrites the replica's entry for id; Apply of a block other than 0 takes the entry for its id
    and answers it.  So an Apply answers exactly when the replica's previous event on that id is a Notify.  Entries
    still in a map at the end of a batch carry over to the next."""

    def __init__(self):
        self.carry = np.zeros(0, FSM_DT)

    def feed(self, raw: bytes) -> np.ndarray:
        ins = np.frombuffer(raw, FSM_DT)
        ev = np.concatenate([self.carry, ins[(ins["kind"] == abi.FSM_NOTIFY) | (ins["id"] != 0)]])
        ev = ev[np.lexsort((np.arange(len(ev)), ev["id"], ev["node"], ev["group"]))]   # per (replica, id), stream order
        same = np.zeros(len(ev), bool)
        same[1:] = (ev["group"][1:] == ev["group"][:-1]) & (ev["node"][1:] == ev["node"][:-1]) & (ev["id"][1:] == ev["id"][:-1])
        notify = ev["kind"] == abi.FSM_NOTIFY
        hit = np.zeros(len(ev), bool)
        hit[1:] = ~notify[1:] & same[1:] & notify[:-1]
        last = np.ones(len(ev), bool)
        last[:-1] = ~same[1:]
        self.carry = ev[last & notify]
        at = np.nonzero(hit)[0]
        out = np.zeros(len(at), RESP_DT)
        out["group"], out["node"], out["id"] = ev["group"][at], ev["node"][at], ev["id"][at]
        out["ckind"], out["cid"], out["tok"] = ev["ckind"][at - 1], ev["cid"][at - 1], ev["data"][at - 1]
        return out    # (group, node, id) order, stream order among equal ids


def response_arrays(runs) -> np.ndarray:
    """The engine's JR_FSMR_RESPONSE runs as RESP_DT rows in (group, node, id) order, stream order among equal ids."""
    rec = np.frombuffer(b"".join(bytes(rc) for rc in runs), np.dtype([("group", "<u4"), ("hdr", "<u4"), ("id0", "<u4"),
                                                                       ("addr", "<u4"), ("tok0", "<u8"), ("stride", "<u8")]))
    cnt = (rec["hdr"] >> 8).astype(np.int64)
    at = np.repeat(np.arange(len(rec)), cnt)
    i = (np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt)).astype(np.uint64)
    out = np.zeros(len(at), RESP_DT)
    out["group"], out["node"] = rec["group"][at], ((rec["hdr"][at] >> 2) & 7) + 1
    out["ckind"], out["cid"] = rec["addr"][at] >> 16, rec["addr"][at] & 0xFFFF
    out["tok"] = rec["tok0"][at] + i * rec["stride"][at]
    out["id"] = rec["id0"][at].astype(np.uint64) + i
    return out[np.lexsort((out["id"], out["node"], out["group"]))]


# ---- the scenario of the GPU suite: isolation, a partition, heal, at any size ------------------------------------------
def partition_scenario(make, G, R, check_every=True, quantum=16):
    """Steady state with auto-truncate and tokens; at quantum k isolate 10% of the leaders and partition {1,2} | {3..5}
    in another 5% of the groups; heal at k + m; continue.  Engine vs oracle and vs a never-folding twin after every
    quantum; returns the fold counts (during the cut, after the heal) and the number of groups with a cut."""
    cfg = dict(seed=21, chain_capacity=128, fsm_units=64)
    eng = make(G, R, flags=CAP | RESP | LINKS, **cfg)
    twin = make(G, R, flags=CAP | RESP | LINKS | NOFOLD, **cfg)
    ora = _oracle(G, R, flags=CAP | LINKS, **cfg)
    apis = (eng, twin, ora)
    cap = G * R * 4 * max(quantum, 24) + 4096
    now = 100
    for api in apis:
        api.step(0, flags=0, inject=bootstrap(G, R))
        api.set_auto_truncate(6)
        api.run(now, 100, 24, 1)
    now += 2400
    ref, answered = ResponseRef(), []

    def drain_and_compare(k):
        want = drain_bytes(ora, cap)
        assert drain_bytes(eng, cap) == want and drain_bytes(twin, cap) == want, k
        re, rt = eng.fsm_responses(), twin.fsm_responses()
        assert re[1].n_dropped == 0 and [bytes(x) for x in re[0]] == [bytes(x) for x in rt[0]], k
        got, exp = response_arrays(re[0]), ref.feed(want)
        assert len(got) == len(exp) and (got == exp).all(), k      # the oracle's Instructions through fsm::Driver
        answered.append(len(got))

    drain_and_compare("bootstrap")
    part_groups = [g for g in range(G) if g % 20 == 3]      # 5%
    cut_groups, folds = None, {}

    def quantum_step(k):
        nonlocal now
        toks = [[((k * quantum + t) << 24 | g) + 1 for g in range(G)] for t in range(quantum)]
        for api in apis:
            api.leader_table()
            api.run_tokens(now, 100, toks)
        now += 100 * quantum
        drain_and_compare(k)
        assert eng.state_digest() == ora.state_digest() == twin.state_digest(), k
        assert eng.leader_table() == ora.leader_table()
        if check_every:
            assert snapshot(eng, G, R) == snapshot(ora, G, R), k

    K, M = 3, 6
    for k in range(K):
        quantum_step(k)
    folds["before"] = eng.fold_count()
    n = [api.isolate_leaders(5, 100) for api in apis]
    assert n[0] == n[1] == n[2] > 0
    iso = {g for g, m in enumerate(eng.links()) if m}
    part_groups = [g for g in part_groups if g not in iso]
    for api in apis:
        api.set_links([partition(R, [1, 2])] * len(part_groups), groups=part_groups)
    links = eng.links()
    assert links == ora.links() == twin.links()
    cut_groups = sum(1 for m in links if m)
    during = []
    for k in range(K, K + M):
        quantum_step(k)
        during.append(eng.fold_count())
        assert eng.fold_count() <= G - cut_groups
    for api in apis:
        api.set_links([0] * G)
    after = []
    for k in range(K + M, K + M + 4):
        quantum_step(k)
        after.append(eng.fold_count())
    assert snapshot(eng, G, R) == snapshot(ora, G, R)
    # an engine that never had a cut, in the same state, folds the same groups
    fresh = make(G, R, flags=CAP | RESP | LINKS, **cfg)
    fresh.restore(eng.save())
    fresh.set_auto_truncate(6)
    toks = [[((1 << 30) + t << 24 | g) + 1 for g in range(G)] for t in range(quantum)]
    for api in (eng, fresh):
        api.run_tokens(now, 100, toks)
    assert fresh.fold_count() == eng.fold_count() and fresh.state_digest() == eng.state_digest()
    after.append(eng.fold_count())
    # the reference's own behaviour (SURVEY N1): an isolated leader's followers never elect, and after the heal the old
    # leader carries on in its term
    assert sum(answered) > G * quantum      # (requests were answered all along, not only compared empty)
    for g in sorted(iso)[:50]:
        assert eng.query(g, 1).role == abi.ROLE_LEADER
    return folds["before"], during, after, cut_groups


def test_partition_scenario_emu():
    G, R = 256, 5
    before, during, after, cut = partition_scenario(_emu, G, R)
    assert before == G and cut > 0
    assert during == [G - cut] * len(during)       # every group without a cut folds, no group with one does
    assert min(after) >= G - cut


# ---- checkpoint and group move -------------------------------------------------------------------------------------------
def _partitioned(make, G, R, **kw):
    cfg = dict(seed=4, flags=CAP | LINKS, chain_capacity=64, fsm_units=96)
    cfg.update(kw)
    api = make(G, R, **cfg)
    api.step(0, flags=0, inject=bootstrap(G, R))
    api.run(100, 100, 8, 0)
    api.set_links([partition(R, [1]), partition(R, [1, 2]), link_cut(R, [(3, 1), (2, 4)])], groups=[2, 5, 9])
    api.leader_table()
    api.run_tokens(900, 100, [[(t << 20) + g + 1 for g in range(G)] for t in range(5)])
    return api


def _checkpoint(make):
    G, R = 40, 5
    a = _partitioned(make, G, R)
    blob = a.save()
    b = make(G, R, seed=4, flags=CAP | LINKS, chain_capacity=64, fsm_units=96)
    b.restore(blob)
    assert b.links() == a.links()
    for api in (a, b):
        api.run(1400, 100, 10, 0)
        api.set_links([0] * G)
        api.run(2400, 100, 12, 0)
    assert a.save() == b.save()
    assert snapshot(a, G, R) == snapshot(b, G, R)


def _move(make):
    G, R = 40, 5
    # the twin never moves; group 5 of `src` (global id 5) moves to slot 2 of `dst` (group_offset 3: global id 5)
    twin, src = _partitioned(make, G, R), _partitioned(make, G, R)
    dst = make(G, R, seed=4, group_offset=3, flags=CAP | LINKS, chain_capacity=64, fsm_units=96)
    cap = G * R * 400
    drain_bytes(twin, cap)
    drain_bytes(src, cap)
    img = src.export_groups([5])
    assert src.links([5]) == twin.links([5])            # the source slot keeps its matrix
    dst.import_groups([2], img)
    assert dst.links([2]) == twin.links([5]) == [partition(R, [1, 2])]
    for api in (twin, dst):
        api.run(1400, 100, 10, 0)
    assert snapshot_group(dst, 2, R) == snapshot_group(twin, 5, R)
    for api in (twin, dst):
        api.set_links([0], groups=[5 if api is twin else 2])
        api.run(2400, 100, 12, 0)
    assert snapshot_group(dst, 2, R) == snapshot_group(twin, 5, R)


def snapshot_group(api, g, R):
    st = [(s.current_term, s.voted_for, s.leader_id, s.election_time_ms, s.election_timeout_ms, s.rng_draws, s.head,
           s.commit, s.id_gen, s.max_key, s.heartbeat_time_ms, tuple(s.progress_head), s.role, s.fault, s.alive,
           s.chain_floor) for s in api.query_many([(g, n) for n in range(1, R + 1)])]
    return st, api.chain_read_many([(g, n, s[15], 40) for n, s in zip(range(1, R + 1), st)])


def test_checkpoint_carries_links_emu():
    _checkpoint(_emu)


def test_group_move_carries_links_emu():
    _move(_emu)


# Without the flag, group images are byte-identical to those of the engine before peer links existed, and checkpoints
# keep their size: the values below were taken from that engine (host build) with this script.
NO_FLAG_IMAGES = {
    3: (1220104, 2816, "72b08062171490ffeb2789a0797d3ae5decc6d411dd800365715d57a977ecf54"),
    5: (2038280, 4704, "8e1633f9ca1d1cce2f472b69cd62d61c85a424b9c2425e72721f91d8297ecb98"),
}


def _no_flag_layout(make):
    import hashlib
    for R, (save_bytes, image_bytes, image_sha) in NO_FLAG_IMAGES.items():
        G = 40
        a = make(G, R, seed=1, flags=CAP | RESP, chain_capacity=48, fsm_units=96)
        b = make(G, R, seed=1, flags=CAP | RESP | LINKS, chain_capacity=48, fsm_units=96)
        for api in (a, b):
            api.step(0, flags=0, inject=bootstrap(G, R))
            api.run(100, 100, 7, 1)
        img = a.export_groups([1, 7])
        assert (len(a.save()), len(img), hashlib.sha256(img).hexdigest()) == (save_bytes, image_bytes, image_sha)
        assert len(b.save()) == save_bytes + 8 * 64      # the flag adds one u64 per group of the padded G, nothing else


def test_checkpoints_and_images_without_flag_keep_their_bytes_emu():
    _no_flag_layout(_emu)


@pytest.mark.gpu
def test_checkpoints_and_images_without_flag_keep_their_bytes_gpu():
    _no_flag_layout(_gpu)


def _reset(make):
    G, R = 40, 5
    api = _partitioned(make, G, R)
    assert any(api.links())
    api._check(api._lib.jr_engine_reset(api._h), "engine_reset")
    assert api.links() == [0] * G                      # fully connected again
    fresh = make(G, R, seed=4, flags=CAP | LINKS, chain_capacity=64, fsm_units=96)
    for x in (api, fresh):
        x.step(0, flags=0, inject=bootstrap(G, R))
        x.run(100, 100, 8, 0)
    assert snapshot(api, G, R) == snapshot(fresh, G, R) and api.fold_count() == fresh.fold_count()


def test_reset_heals_every_link_emu():
    _reset(_emu)


@pytest.mark.gpu
def test_reset_heals_every_link_gpu():
    _reset(_gpu)


@pytest.mark.parametrize("make", [_emu, _oracle], ids=["emu", "oracle"])
def test_isolate_counts_leaders_with_nothing_to_cut(make):
    """R = 1: a leader has no link, so nothing is cut, yet each picked group with a live leader counts."""
    G = 64
    a, b = make(G, 1, seed=3, flags=LINKS), make(G, 1, seed=3, flags=LINKS)
    for api in (a, b):
        api.step(0, flags=0, inject=bootstrap(G, 1))
    n = a.isolate_leaders(9, 500)
    assert n == b.kill_leaders(9, 500) > 0
    assert a.links() == [0] * G


# ---- a long partition with truncation: the majority's leader runs out of window, as in the oracle ------------------------
def _long_partition(make):
    G, R = 40, 5
    cfg = dict(seed=6, flags=CAP | LINKS, chain_capacity=16, fsm_units=96)
    eng, ora = make(G, R, **cfg), _oracle(G, R, **cfg)
    first = {}
    for api in (eng, ora):
        api.step(0, flags=0, inject=bootstrap(G, R))
        api.set_auto_truncate(2)
        api.run(100, 100, 8, 1)
        api.set_links([partition(R, [5])] * G)          # a follower cut off: alive, it holds every floor down
    for t in range(60):
        for api in (eng, ora):
            api.run(900 + 100 * t, 100, 1, 1)
            api.discard_fsm(strict=False)
        fe, fo = eng.fault_count(), ora.fault_count()
        assert fe == fo, t
        assert eng.state_digest() == ora.state_digest(), t
        if fe and "t" not in first:
            first["t"] = t
    assert "t" in first
    st = eng.query(0, 1)
    assert st.fault == abi.FAULT_ENGINE_CHAIN_CAPACITY and st.role == abi.ROLE_LEADER
    assert snapshot(eng, G, R) == snapshot(ora, G, R)


def test_long_partition_faults_like_oracle_emu():
    _long_partition(_emu)


# ---- on the H100 ---------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_partition_scenario_gpu_65536():
    G, R = 65536, 5
    before, during, after, cut = partition_scenario(_gpu, G, R, check_every=False)
    assert before == G and cut > G // 10
    assert during == [G - cut] * len(during)
    assert min(after) >= G - cut


@pytest.mark.gpu
def test_checkpoint_carries_links_gpu():
    _checkpoint(_gpu)


@pytest.mark.gpu
def test_group_move_carries_links_gpu():
    _move(_gpu)


@pytest.mark.gpu
def test_long_partition_faults_like_oracle_gpu():
    _long_partition(_gpu)


@pytest.mark.gpu
def test_random_scripts_gpu():
    for R in (3, 5, 7):
        G = 40
        rng = random.Random(7 * R)
        cfg = dict(seed=R, chain_capacity=48, fsm_units=96, mailbox_units=128)   # (lagging followers of R = 7: many AppendEntries runs)
        eng, ora = _gpu(G, R, flags=CAP | LINKS, **cfg), _oracle(G, R, flags=CAP | LINKS, **cfg)
        ce, co, cap = Clock(), Clock(), G * R * 400
        for i, call in enumerate(random_calls(rng, G, R, 36)):
            assert play(eng, G, R, call, ce) == play(ora, G, R, call, co), (R, i)
            assert eng.links() == ora.links() and eng.state_digest() == ora.state_digest(), (R, i)
            assert snapshot(eng, G, R) == snapshot(ora, G, R), (R, i)
            assert drain_bytes(eng, cap) == drain_bytes(ora, cap), (R, i)


# ---- the two restatements, differenced with cuts ---------------------------------------------------------------------------
@pytest.mark.parametrize("R", [3, 5])
def test_python_restatement_agrees_with_cuts(R):
    """The C++ oracle's cut delivery (links.cpp) against the same filter on the independent Python restatement, step by
    step: every emitted Message, every Instruction, every replica's state."""
    from tests.oracle_links.links import PyLinkCluster
    from josefine_b200.raft import msg_tuple
    G = 6
    cfg = dict(seed=30 + R, chain_capacity=64, flags=abi.F_CAPTURE_MESSAGES | CAP | LINKS)
    a, b = _oracle(G, R, **cfg), PyLinkCluster.create(G, R, **cfg)
    rng = random.Random(R)
    for api in (a, b):
        api.step(0, flags=0, inject=bootstrap(G, R))
    for t in range(1, 120):
        if t % 15 == 0:
            gs = rng.sample(range(G), 3)
            cuts = [rng.choice([0, partition(R, rng.sample(range(1, R + 1), R // 2)),
                                rng.getrandbits(64) & valid_mask(R) & rng.getrandbits(64)]) for _ in gs]
            for api in (a, b):
                api.set_links(cuts, groups=gs)
        inj = [Command.client_request(g, rng.randint(1, R), t * 100 + g) for g in range(G) if rng.random() < 0.3]
        if t % 23 == 0:
            inj.append(Command.timeout(rng.randrange(G), rng.randint(1, R)))
        ra, rb = a.step(100 * t, inject=inj), b.step(100 * t, inject=inj)
        assert [msg_tuple(m) for m in ra.messages] == [msg_tuple(m) for m in rb.messages], t
        assert [fsm_tuple(f) for f in ra.fsm] == [fsm_tuple(f) for f in rb.fsm], t
        for g in range(G):
            for n in range(1, R + 1):
                sa, sb = a.query(g, n), b.query(g, n)
                assert (sa.current_term, sa.role, sa.head, sa.commit, sa.fault, sa.leader_id, sa.voted_for) == \
                       (sb.current_term, sb.role, sb.head, sb.commit, sb.fault, sb.leader_id, sb.voted_for), (t, g, n)
    assert a.links() == b.links()
