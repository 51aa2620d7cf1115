"""Group export and import (jr_group_export / jr_group_import): Raft groups leave one engine with their mail in flight and
their undrained Instructions and run on in another engine, another slot, or the same one.  Every case runs on the device
code (CPU emulation) and on the GPU.  Moves happen at moments when each carried item is non-trivial: mid-election,
leaders in Probe, client requests queued on leaderless followers, mail right after AppendEntries, a non-zero floor,
pending restart marks, unmatched Notifies, an announced route, with and without stream digests."""
import ctypes as C

import pytest

from josefine_b200 import abi, Command, RaftError
from josefine_b200.raft import expand_responses
from tests.golden_scenarios import bootstrap

CAP, RESP, DIG = abi.F_CAPTURE_FSM, abi.F_CLIENT_RESPONSES, abi.F_STREAM_DIGEST


def _oracle(g, r, **kw):
    from tests.oracle_move.movable import MovableCluster
    return MovableCluster.create(g, r, n_threads=16 if g >= 1024 else 1, **kw)


def _emu(g, r, **kw):
    from tests.emu.emu import EmuEngine
    return EmuEngine.create(g, r, **kw)


def _gpu(g, r, **kw):
    from josefine_b200 import RaftEngine
    return RaftEngine.create(g, r, **kw)


def _cfg(digest, seed=5, offset=0):
    return dict(seed=seed, group_offset=offset, flags=CAP | RESP | (DIG if digest else 0), chain_capacity=64, fsm_units=96)


# ---- the batched drain, one call at a time (three batches may be outstanding) ---------------------------------------
def rec_async(api):
    api._check(api._fn("fsm_records_async")(api._h), "fsm_records_async")


def rec_wait(api):
    """The oldest outstanding batch: its records (bytes) and the responses the drain produced (bytes)."""
    ptr, batch = C.POINTER(abi.FsmRecord)(), abi.FsmBatch()
    api._check(api._fn("fsm_records_wait")(api._h, C.byref(ptr), C.byref(batch)), "fsm_records_wait")
    recs = [bytes(ptr[i]) for i in range(batch.n_records)]
    runs, rb = api.fsm_responses()
    assert rb.n_dropped == 0
    return recs, [bytes(x) for x in runs]


def _tokens(G, k, base):
    return [[(base + 1000 * t + g) if (g + t) % 3 else 0 for g in range(G)] for t in range(k)]


# ---- one script of calls; `hook(i)` runs between call i - 1 and call i -----------------------------------------------
def script(api, G, R, hook, out, synth=1):
    """Every call shape: jr_step with injects, fused runs the fold takes, run_tokens after an announce, async drains with
    three batches outstanding, restarts with their marks pending, truncation.  Appends every output to `out`.  synth=0:
    no synthetic proposals (their tokens carry the engine's step index, which a move to another engine changes)."""
    half = [g for g in range(G) if g % 2]
    pending = []   # the engines the outstanding batches were enqueued on, oldest first

    def enqueue():
        pending.append(getattr(api, "target", api))
        rec_async(pending[-1])

    calls = [
        # client requests on leaderless followers: queued (follower.rs:258-270)
        lambda: api.step(0, flags=0, inject=[Command.client_request(g, 2, 7000 + g) for g in half]),
    ]
    # plain ticks: the election timers (500-1000 ms) fire, candidates collect votes, leaders start in Probe
    calls += [(lambda k=k: api.step(100 * k)) for k in range(1, 13)]
    calls += [
        lambda: out.append(("lt", api.leader_table())),
        lambda: api.run_tokens(1300, 100, _tokens(G, 3, 1 << 40)),          # route announced, then proposals
        enqueue,
        lambda: api.run(1600, 100, 1, 2 * synth),                                    # AppendEntries in flight
        enqueue,
        lambda: api.node_restart_many(1700, [(g, 2, None, 0, None) for g in range(0, G, 3)]),   # restart marks pending
        lambda: api.run_tokens(1700, 100, _tokens(G, 2, 2 << 40)),          # Notifies not yet matched
        enqueue,
        lambda: out.append(("b", rec_wait(pending.pop(0)))),
        lambda: api.set_auto_truncate(4),
        lambda: api.run(1900, 100, 12, synth),                                   # the fold, truncation
        lambda: out.append(("b", rec_wait(pending.pop(0)))),
        lambda: out.append(("b", rec_wait(pending.pop(0)))),
        lambda: api.run(3100, 100, 2, synth),                                    # mail right after a fused run
        lambda: out.append(("lt", api.leader_table())),
        lambda: api.run_tokens(3300, 100, _tokens(G, 4, 3 << 40)),
        lambda: out.append(("fold", api.fold_count())),
        lambda: api.run(3700, 100, 9, synth),
        enqueue,
        lambda: out.append(("b", rec_wait(pending.pop(0)))),
    ]
    for i, c in enumerate(calls):
        hook(i)
        c()
    hook(len(calls))
    return len(calls)


N_CALLS = 33


def snapshot(api, G, R, groups=None):
    groups = range(G) if groups is None else groups
    tg = [(g, n) for g in groups for n in range(1, R + 1)]
    st = [(s.current_term, s.voted_for, s.leader_id, s.election_time_ms, s.election_timeout_ms, s.rng_draws, s.head,
           s.commit, s.id_gen, s.max_key, s.heartbeat_time_ms, s.votes_seen, s.votes_granted, tuple(s.progress_head),
           s.progress_replicate, s.role, s.fault, s.alive, s.n_queued, s.chain_floor) for s in api.query_many(tg)]
    reqs = [(g, n, s[19], 40) for (g, n), s in zip(tg, st)]
    return st, api.chain_read_many(reqs)


def full_compare(a, b, G, R, digest):
    assert a.state_digest() == b.state_digest()
    assert a.fault_count() == b.fault_count()
    if digest:
        assert a.stream_digest() == b.stream_digest()
    assert snapshot(a, G, R) == snapshot(b, G, R)


# ---- 1. round trip is invisible ---------------------------------------------------------------------------------------
def case_round_trip(make, at, digest, R=3, G=40):
    a, b = make(G, R, **_cfg(digest)), make(G, R, **_cfg(digest))
    groups = [g for g in range(G) if g % 4 != 1]
    oa, ob = [], []

    def hook(i):
        if i == at:
            img = a.export_groups(groups)
            a.import_groups(groups, img)

    n = script(a, G, R, hook, oa)
    script(b, G, R, lambda i: None, ob)
    assert n == N_CALLS
    assert oa == ob
    if not digest:   # (the stream digests keep every launch off the fold)
        assert any(k == "fold" and v > 0 for k, v in oa), "the fold must take groups in the script"
    full_compare(a, b, G, R, digest)


MOMENTS = [1, 7, 11, 14, 17, 19, 21, 24, 27, 30, 32]   # queued requests, mid-election, Probe, ... (see `script`)


@pytest.mark.parametrize("at", MOMENTS)
@pytest.mark.parametrize("digest", [False, True])
def test_round_trip_is_invisible_on_device_code(at, digest):
    case_round_trip(_emu, at, digest)


@pytest.mark.gpu
@pytest.mark.parametrize("at", MOMENTS)
@pytest.mark.parametrize("digest", [False, True])
def test_round_trip_is_invisible_on_gpu(at, digest):
    case_round_trip(_gpu, at, digest)


def test_moments_are_non_trivial_on_device_code():
    """The moments the round trips export at hold what they are meant to: queued requests, candidates with votes,
    leaders in Probe, a non-zero floor."""
    G, R = 40, 3
    api = _emu(G, R, **_cfg(False))
    seen = {}

    def hook(i):
        if i not in MOMENTS:
            return
        st = api.query_many([(g, n) for g in range(G) for n in range(1, R + 1)])
        seen[i] = dict(cand=sum(s.role == abi.ROLE_CANDIDATE and s.votes_seen != 0 for s in st),
                       probe=sum(s.role == abi.ROLE_LEADER and s.progress_replicate != (1 << R) - 1 for s in st),
                       queued=sum(s.n_queued for s in st), floor=max(s.chain_floor for s in st))
    script(api, G, R, hook, [])
    assert seen[1]["queued"] > 0
    assert any(v["cand"] for v in seen.values()) and any(v["probe"] for v in seen.values())
    assert any(v["floor"] > 0 for v in seen.values())


# ---- 2. another engine, the same global ids ---------------------------------------------------------------------------
def case_other_engine(make, at, pre, G=40, R=3):
    cfg = _cfg(True)
    twin, c = make(G, R, **cfg), make(G, R, **cfg)
    for k in range(pre):   # pre odd: the destination's mailbox parity differs from the source's at every moment
        c.step(0)
    groups = [g for g in range(G) if g % 3]
    ot, oc = [], []
    a = make(G, R, **cfg)
    state = {"api": a}

    class Switch:   # the source takes the calls up to the move, the destination takes the rest
        target = property(lambda self: state["api"])

        def __getattr__(self, name):
            return getattr(state["api"], name)

    def hook(i):
        if i == at:
            c.import_groups(groups, a.export_groups(groups))
            state["api"] = c
            if at > 22:   # an engine setting, not group state: the destination runs with the source's
                c.set_auto_truncate(4)

    script(Switch(), G, R, hook, oc, synth=0)
    script(twin, G, R, lambda i: None, ot, synth=0)
    assert snapshot(c, G, R, groups) == snapshot(twin, G, R, groups)
    # the union of the source's batches before the move and the destination's after it: the twin's, for these groups
    mine = set(groups)

    def of(out):
        recs, resp = [], []
        for k, v in out:
            if k == "b":
                recs += [r for r in v[0] if abi.FsmRecord.from_buffer_copy(r).group in mine]
                resp += [r for r in v[1] if abi.FsmRecord.from_buffer_copy(r).group in mine]
        return sorted(recs), sorted(resp)
    assert of(oc) == of(ot)
    lt_c = [v for k, v in oc if k == "lt"]
    lt_t = [v for k, v in ot if k == "lt"]
    assert [[x[g] for g in groups] for x in lt_c] == [[x[g] for g in groups] for x in lt_t]


@pytest.mark.parametrize("at", [7, 17, 21, 27])
@pytest.mark.parametrize("pre", [1, 2])
def test_move_to_another_engine_on_device_code(at, pre):
    case_other_engine(_emu, at, pre)


@pytest.mark.gpu
@pytest.mark.parametrize("at", [7, 17, 21, 27])
@pytest.mark.parametrize("pre", [1, 2])
def test_move_to_another_engine_on_gpu(at, pre):
    case_other_engine(_gpu, at, pre)


# ---- 3. other slots, another group_offset and seed, a permutation: against the oracle --------------------------------
def _continue(api, G, now):
    out = []
    api.run(now, 100, 6, 1)
    out.append(api.leader_table())
    api.run_tokens(now + 600, 100, _tokens(G, 3, 9 << 40))
    api.step(now + 900)
    api.run(now + 1000, 100, 20, 1)
    out.append([(f.group, f.node, f.kind, f.client_kind, f.client_id, f.block.id, f.block.next, f.block.data)
                for f in api.drain_fsm(cap=1 << 18)])
    out.append(api.leader_table())
    return out


def _prelude(api, G, R):
    api.step(0, flags=0, inject=bootstrap(G, R))
    api.set_auto_truncate(4)
    api.run(100, 100, 8, 1)
    api.leader_table()
    api.run_tokens(900, 100, _tokens(G, 2, 1 << 40))
    api.step(1100, flags=abi.STEP_DELIVER | abi.STEP_TICK | abi.STEP_SYNTH_PROPOSALS, n_synth=1)


def case_against_oracle(make, R=3):
    G1, G2 = 24, 40
    c1, c2 = dict(_cfg(True, seed=3, offset=0)), dict(_cfg(True, seed=11, offset=1000))
    for c in (c1, c2):
        c["flags"] = CAP | DIG
    e1, e2, o1, o2 = make(G1, R, **c1), make(G2, R, **c2), _oracle(G1, R, **c1), _oracle(G2, R, **c2)
    for api, G in ((e1, G1), (e2, G2), (o1, G1), (o2, G2)):
        _prelude(api, G, R)
    e2.step(1200)
    o2.step(1200)   # another mailbox parity
    groups, slots = [3, 0, 17, 9, 22], [39, 5, 6, 0, 21]
    e2.import_groups(slots, e1.export_groups(groups))
    o1.group_move(o2, groups, slots)
    perm_from, perm_to = [1, 2, 4, 8], [8, 1, 2, 4]          # a permutation within one engine
    e1.import_groups(perm_to, e1.export_groups(perm_from))
    o1.group_move(o1, perm_from, perm_to)
    for (e, o, G) in ((e1, o1, G1), (e2, o2, G2)):
        assert e.state_digest() == o.state_digest()
        assert _continue(e, G, 1300) == _continue(o, G, 1300)
        assert e.state_digest() == o.state_digest()
        assert e.stream_digest() == o.stream_digest()
        assert e.fault_count() == o.fault_count() == 0
        assert snapshot(e, G, R) == snapshot(o, G, R)


def test_against_the_oracle_on_device_code():
    case_against_oracle(_emu)


@pytest.mark.gpu
def test_against_the_oracle_on_gpu():
    case_against_oracle(_gpu, R=5)


# ---- 4. exactly once --------------------------------------------------------------------------------------------------
def case_exactly_once(make, G=16, R=3):
    cfg = _cfg(False)
    src, dst = make(G, R, **cfg), make(G, R, **cfg)
    src.step(0, flags=0, inject=bootstrap(G, R))
    src.run(100, 100, 10, 0)
    src.leader_table()
    src.discard_fsm()
    src.run_tokens(1100, 100, [[0xabc00 + g for g in range(G)]])   # proposed (Notify emitted), not yet committed
    rec_async(src)                                                 # a batch outstanding across the export
    img = src.export_groups(range(G))
    recs0, resp0 = rec_wait(src)
    dst.import_groups(range(G), img)
    dst.run(1200, 100, 6, 0)
    rec_async(dst)
    recs1, resp1 = rec_wait(dst)
    rec_async(src)
    recs2, resp2 = rec_wait(src)
    assert recs2 == [] and resp2 == []                             # the detached source drains nothing more
    notifies = lambda rs: sum(abi.FsmRecord.from_buffer_copy(r).hdr & 3 == abi.FSMR_NOTIFY for r in rs)  # noqa: E731
    answers = expand_responses([abi.FsmRecord.from_buffer_copy(r) for r in resp0 + resp1])
    toks = sorted(x[3] for x in answers)
    assert toks == sorted(0xabc00 + g for g in range(G)), "each request answered exactly once"
    assert resp0 == [] and notifies(recs0) == G and notifies(recs1) == 0


def test_exactly_once_on_device_code():
    case_exactly_once(_emu)


@pytest.mark.gpu
def test_exactly_once_on_gpu():
    case_exactly_once(_gpu)


# ---- 5. detach --------------------------------------------------------------------------------------------------------
def case_detach(make, G=16, R=3):
    api = make(G, R, **_cfg(True))
    api.step(0, flags=0, inject=bootstrap(G, R))
    api.run(100, 100, 10, 1)
    gone = [2, 5, 11]
    before = snapshot(api, G, R, gone)
    img = api.export_groups(gone)
    after = snapshot(api, G, R, gone)
    assert all(s[17] == 0 for s in after[0])
    assert [s[:17] + s[18:] for s in after[0]] == [s[:17] + s[18:] for s in before[0]] and after[1] == before[1]
    n0 = api.stream_digest()
    api.run(1100, 100, 10, 1)
    recs = [abi.FsmRecord.from_buffer_copy(r) for r in api.fsm_records()[0]]
    assert not any(r.group in gone for r in recs)
    assert snapshot(api, G, R, gone) == after            # inert: nothing steps, nothing is emitted
    assert api.stream_digest()[2] > n0[2]
    api.import_groups(gone, img)                         # an import over a detached slot brings it back
    assert all(s[17] == 1 for s in snapshot(api, G, R, gone)[0])
    api.run(2100, 100, 4, 1)
    recs = [abi.FsmRecord.from_buffer_copy(r) for r in api.fsm_records()[0]]
    assert set(gone) <= {r.group for r in recs}


def test_detach_on_device_code():
    case_detach(_emu)


@pytest.mark.gpu
def test_detach_on_gpu():
    case_detach(_gpu)


# ---- 6. refusals leave the engine untouched ---------------------------------------------------------------------------
def _refused(api, fn):
    d0, s0 = api.state_digest(), api.save()
    with pytest.raises(RaftError) as ei:
        fn()
    assert ei.value.status == abi.E_INVAL
    assert api.state_digest() == d0 and api.save() == s0


def case_refusals(make, G=8, R=3):
    cfg = _cfg(False)
    src = make(G, R, **cfg)
    src.step(0, flags=0, inject=bootstrap(G, R))
    src.run(100, 100, 6, 1)
    img = src.export_groups([1, 2, 3])
    dst = make(G, R, **cfg)
    dst.run(100, 100, 3, 0)
    for field, value in [("n_replicas", 5), ("chain_capacity", 128), ("mailbox_units", 96), ("fsm_units", 32),
                         ("election_min_ms", 400), ("election_max_ms", 1200), ("heartbeat_ms", 50),
                         ("resident_mask", 3), ("flags", CAP)]:
        other = make(G, value, **cfg) if field == "n_replicas" else make(G, R, **{**cfg, field: value})
        _refused(other, lambda: other.import_groups([1, 2, 3], img))
    ok = make(G + 8, R, **{**cfg, "seed": 99, "group_offset": 7, "flags": cfg["flags"] | abi.F_NO_SYMMETRIC_FOLD})
    ok.import_groups([9, 0, 4], img)                      # the fields that may differ
    bad = bytearray(img)
    bad[0] ^= 1
    _refused(dst, lambda: dst.import_groups([1, 2, 3], bytes(bad)))          # magic
    for pos in (40, 200, len(img) // 2, len(img) - 1):                     # one flipped byte: the checksum
        bad = bytearray(img)
        bad[pos] ^= 0x10
        _refused(dst, lambda: dst.import_groups([1, 2, 3], bytes(bad)))
    _refused(dst, lambda: dst.import_groups([1, 2, 3], img[:-16]))          # truncated
    _refused(dst, lambda: dst.import_groups([1, 2, 3], img[:64]))
    _refused(dst, lambda: dst.import_groups([1, 2], img))                   # n mismatch
    _refused(dst, lambda: dst.import_groups([1, 2, G], img))                # slot out of range
    _refused(dst, lambda: dst.import_groups([1, 2, 1], img))                # slot named twice
    _refused(src, lambda: src.export_groups([4, 5, 4]))                     # group named twice
    _refused(src, lambda: src.export_groups([4, G]))                        # group out of range
    # a capacity-sizing call does not detach
    d0, s0 = src.state_digest(), src.save()
    need = C.c_size_t(0)
    gs = (C.c_uint32 * 2)(4, 5)
    assert src._fn("group_export")(src._h, gs, C.c_size_t(2), None, C.c_size_t(0), C.byref(need)) == abi.E_CAPACITY
    buf = C.create_string_buffer(need.value)
    assert src._fn("group_export")(src._h, gs, C.c_size_t(2), buf, C.c_size_t(need.value - 1), C.byref(need)) == abi.E_CAPACITY
    assert src.state_digest() == d0 and src.save() == s0


def test_refusals_on_device_code():
    case_refusals(_emu)


@pytest.mark.gpu
def test_refusals_on_gpu():
    case_refusals(_gpu)


# ---- 7. full size -----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_full_size_move_65536x5():
    """65,536 x 5, chain_capacity 512, auto-truncate 8: every group moves from one engine into another mid-run, then 256
    more ticks -- the destination equals a never-moved twin and the oracle."""
    G, R = 65536, 5
    cfg = dict(seed=1, chain_capacity=512)
    src, twin, ora = _gpu(G, R, **cfg), _gpu(G, R, **cfg), _oracle(G, R, **cfg)
    dst = _gpu(G, R, **cfg)
    dst.step(0)
    dst.run(100, 100, 128, 0)   # the source's step index: synthetic proposal tokens carry the engine's
    for api in (src, twin, ora):
        api.step(0, flags=0, inject=bootstrap(G, R))
        api.set_auto_truncate(8)
        api.run(100, 100, 64, 1)
        api.run(6500, 100, 64, 1)
    assert src.fold_count() == G   # moved mid-run: out of the symmetric-group fold's steady state
    dst.set_auto_truncate(8)
    dst.import_groups(range(G), src.export_groups(range(G)))
    for api in (dst, twin, ora):
        for k in range(4):
            api.run(12900 + 6400 * k, 100, 64, 1)
    assert dst.state_digest() == twin.state_digest() == ora.state_digest()
    assert dst.leader_table() == twin.leader_table() == ora.leader_table()
    assert dst.fault_count() == 0 and dst.fold_count() == G
    sample = range(0, G, 4099)
    assert snapshot(dst, G, R, sample) == snapshot(ora, G, R, sample)
