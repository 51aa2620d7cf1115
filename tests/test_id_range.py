"""Block ids at the top of the device's 31-bit range (deviation D4), engine against oracle.

Every other parity test starts from a fresh engine, so its ids stay far below 2^31.  Truncation (D7) lets an engine run
forever and makes large ids routine, so here a live cluster is moved to a high base on both sides by the same
order-preserving map, f(v) = v + K for v >= F (F = the group's floor, > 0) and f(v) = v below it: f keeps every order,
equality and the literal 0, and commutes with everything Raft does with ids, so the shifted cluster's future is the
original's future shifted by f, until an id would reach 2^31.  The oracle shifts itself (jro_shift_ids); the engine is
shifted by editing a jr_engine_save checkpoint.  Both shifts happen between steps with no mail in flight and nothing
undrained.  From there the fused calls, truncation, compaction, leader kills with re-election, export and bulk restart
run on both sides and everything observable is compared after every call.  Three bases: the middle of the range with the
table rows moved (a), a window that straddles 2^31 (b), and leaders that append until the id 2^31 faults them (c).

The boundary tests check that ABI input past the limit is refused with the engine untouched."""
import ctypes as C

import numpy as np
import pytest

from josefine_b200 import abi, expand_responses, fsm_tuple
from josefine_b200.verify import verify_groups as verify_restated
from tests.stream_cases import _bootstrap
from tests.test_bulk_restart import _restart_raw
from tests.test_client_responses import DriverRef
from tests.test_sym_entry import Checkpoint

LIMIT = 1 << 31                     # JR_BLOCK_ID_LIMIT
ABSENT = 0xFFFFFFFF
CAP = abi.F_CAPTURE_FSM
HB, DT, SPREAD = 250, 100, 8        # heartbeat, tick; group g's leader is g % SPREAD ids behind the top at the shift
CFG = dict(chain_capacity=100, heartbeat_ms=HB, mailbox_units=64, fsm_units=256)     # rows = 128
KINDS = ("fold", "nofold", "responses")


def _oracle(g, r, **kw):
    from oracle.restated import RestatedCluster
    return RestatedCluster.create(g, r, **kw)


def _emu(g, r, **kw):
    from tests.emu.emu import EmuEngine
    return EmuEngine.create(g, r, **kw)


def _gpu(g, r, **kw):
    from josefine_b200 import RaftEngine
    return RaftEngine.create(g, r, **kw)


def _create(make, kind, G, R, monkeypatch, **cfg):
    """fold: folds; nofold: JR_NO_FOLD=1 and stream digests; responses: F_CLIENT_RESPONSES."""
    flags = CAP | {"nofold": abi.F_STREAM_DIGEST, "responses": abi.F_CLIENT_RESPONSES}.get(kind, 0)
    env = {"nofold": "JR_NO_FOLD"}.get(kind)
    if env:
        monkeypatch.setenv(env, "1")
    api = make(G, R, flags=flags, **cfg)
    if env:
        monkeypatch.delenv(env)
    api.kind, api.cfg_dict = kind, dict(cfg, flags=flags)
    return api


# ---- the engine's shift: a jr_engine_save checkpoint edited in place ---------------------------------------------------

def shift_engine(api, K):
    """Apply f to every id in api's checkpoint and restore it: P2 head / commit / id_gen, MK, TB, a leader's progress
    heads, the non-ABSENT CNEXT values, with F_CLIENT_RESPONSES the pending notification runs; the CNEXT / CTOK rows move
    by K mod rows.  Only from a quiet state: no mail in either outbox, every Instruction FIFO drained."""
    G, R = api.n_groups, api.n_replicas
    ck = Checkpoint(api.save(), G, R, api.cfg_dict)
    in_flight, spent = (ck.oc1, ck.oc0) if ck.cur == 0 else (ck.oc0, ck.oc1)
    assert not in_flight.any(), "mail in flight"
    spent[:] = 0                        # the mail the last step consumed: never read again, and it names old ids
    assert not ck.fc.any(), "undrained Instructions"
    Gp = ck.Gp
    floor = np.full(Gp, 1 << 40, np.int64)                     # padding lanes are never shifted
    floor[:G] = ck.tb[:G]
    assert (floor[:G] > 0).all(), "f keeps 0 only above a floor > 0"

    def f(a, where=True):                                       # a: [..., Gp] views; ids at or above the floor move
        v = a.astype(np.int64)
        moved = (v >= floor) & (v != ABSENT) & where
        out = np.where(moved, v + K, v)
        assert (out[moved] < LIMIT).all(), "K takes an id to 2^31"
        a[...] = out.astype(np.uint32)

    p2 = ck.p2.reshape(R, Gp, 4)
    f(p2[:, :, 0]), f(p2[:, :, 1]), f(p2[:, :, 2])             # (views: written through)
    f(ck.mk.reshape(R, Gp))
    leader = (p2[:, :, 3] & 255) == abi.ROLE_LEADER
    pr = ck.pr.reshape(-1, R, Gp, 4)
    for q in range(pr.shape[0]):
        for j in range(4):
            f(pr[q, :, :, j], leader)
    f(ck.tb)
    cn = ck.cnext.reshape(ck.rows, R, Gp)
    f(cn)
    cn[...] = np.roll(cn, K % ck.rows, axis=0)
    ct = ck.ctok.reshape(ck.rows, R, Gp)
    ct[...] = np.roll(ct, K % ck.rows, axis=0)
    if hasattr(ck, "pn"):
        pn = ck.pn.reshape(2 * abi.NOTIFY_RUNS, R, Gp, 4)
        held = ck.pnc[:R * Gp].reshape(R, Gp)
        for k in range(abi.NOTIFY_RUNS):
            live = held > k
            id0, cnt = pn[2 * k, :, :, 0], pn[2 * k, :, :, 1].astype(np.int64)
            lo = id0.astype(np.int64)
            assert not (live & (lo < floor) & (lo + cnt - 1 >= floor)).any(), "a pending run straddles the floor"
            f(id0, live)
    api.restore(bytes(ck.buf))


# ---- comparison -------------------------------------------------------------------------------------------------------

def _records(api):
    """The batched drain, expanded; no APPLY / NOTIFY record may name an id at or past 2^31."""
    recs, batch = api.fsm_records()
    assert batch.n_dropped == 0
    for rc in recs:
        kind, count = rc.hdr & 3, rc.hdr >> 8
        if kind in (abi.FSMR_APPLY, abi.FSMR_NOTIFY):
            assert rc.id0 + count - 1 < LIMIT, f"record names id {rc.id0 + count - 1}"
            if kind == abi.FSMR_APPLY and count == 1:
                assert (rc.stride & 0xFFFFFFFF) < LIMIT
    return recs, api.fsm_expand(recs)


def _fold_check(api, recs, want):
    """jr_fsm_fold / jr_fsm_fold_mt over the batch: the watermark and counts the oracle's Instructions give."""
    G, R = api.n_groups, api.n_replicas
    arr = (abi.FsmRecord * max(len(recs), 1))(*recs)
    for name, extra in (("jr_fsm_fold", ()), ("jr_fsm_fold_mt", (C.c_uint32(3),))):
        hi, tot = np.zeros(R * G, np.uint32), np.zeros(3, np.uint64)
        st = getattr(api._lib, name)(C.cast(arr, C.c_void_p), C.c_size_t(len(recs)), G, R, hi.ctypes.data, tot.ctypes.data,
                                     *extra)
        assert st == abi.OK
        exp_hi = np.zeros(R * G, np.uint32)
        for (g, n, kind, _, _, bid, _, _) in want:
            if kind == abi.FSM_APPLY:
                exp_hi[(n - 1) * G + g] = max(exp_hi[(n - 1) * G + g], bid)
        assert np.array_equal(hi, exp_hi), name
        assert int(tot[0]) == sum(w[2] == abi.FSM_APPLY for w in want) and int(tot[1]) == sum(w[2] == abi.FSM_NOTIFY for w in want)


def _verify(result):
    rep, fnd = result
    fields = lambda x: tuple(getattr(x, f) for f, _ in x._fields_)     # noqa: E731
    return fields(rep), [fields(x) for x in fnd]


class Cluster:
    """Engines of every KIND and the oracle, driven by the same calls and compared after each one."""

    def __init__(self, make, G, R, monkeypatch, seed=7, sample=1, **over):
        cfg = dict(CFG, seed=seed, fsm_host_records=G * R * 64, **over)
        self.G, self.R, self.sample = G, R, sample       # states, windows and verification: every sample-th group
        self.engs = [_create(make, k, G, R, monkeypatch, **cfg) for k in KINDS]
        self.ora = _oracle(G, R, flags=CAP | abi.F_STREAM_DIGEST, n_threads=8 if G > 1000 else 1, **cfg)
        self.ora.kind = "oracle"
        self.ref = DriverRef()                                # fsm::Driver over the oracle's Instructions
        self.now = 0
        self.fold_counts = []

    @property
    def apis(self):
        return self.engs + [self.ora]

    def call(self, name, *args):
        res = [getattr(api, name)(*args) for api in self.apis]
        assert all(r == res[0] for r in res), f"{name}{args}: {res}"
        return res[0]

    def launch(self, name, n, *args):
        for api in self.apis:
            getattr(api, name)(self.now + DT, DT, *args)
        self.now += DT * n
        self.fold_counts.append(self.engs[0].fold_count())
        self.check()

    def check(self, drain=True):
        if drain:
            ins = self.ora.drain_fsm(cap=1 << 22)
            want = [fsm_tuple(i) for i in ins]
            responses = self.ref.feed(ins)
            for e in self.engs:
                recs, got = _records(e)
                assert [fsm_tuple(i) for i in got] == want, f"{e.kind}: Instruction streams differ"
                if e.kind == "fold":
                    _fold_check(e, recs, want)
                if e.kind == "responses":
                    runs, batch = e.fsm_responses()
                    assert batch.n_dropped == 0 and expand_responses(runs) == responses
        G, R = self.G, self.R
        groups = list(range(0, G, self.sample))
        targets = [(g, n) for g in groups for n in range(1, R + 1)]
        st = [[tuple(sorted(s.as_dict().items())) for s in api.query_many(targets)] for api in self.apis]
        for s, api in zip(st[1:], self.apis[1:]):
            assert s == st[0], f"{api.kind}: replica state differs"
        reqs = [(g, n, int(self.ora.query(g, n).chain_floor), self.ora.cfg.chain_capacity) for g, n in targets]
        w = self.ora.chain_read_many(reqs)
        for e in self.engs:
            assert e.chain_read_many(reqs) == w, f"{e.kind}: block windows differ"
        dig, lt, fc = self.ora.state_digest(), self.ora.leader_table(), self.ora.fault_count()
        for e in self.engs:
            assert (e.state_digest(), e.leader_table(), e.fault_count()) == (dig, lt, fc), e.kind
        assert self.engs[KINDS.index("nofold")].stream_digest() == self.ora.stream_digest()
        findings = _verify(verify_restated(self.ora, groups))
        for e in self.engs:
            assert _verify(e.verify_groups(groups)) == findings, f"{e.kind}: jr_verify_groups"
            assert _verify(verify_restated(e, groups)) == findings, f"{e.kind}: verify.py"

    def shift(self, K):
        for e in self.engs:
            shift_engine(e, K)
        self.ora.shift_ids(K)
        self.ref.maps = {key: {(b + K if b >= self.floor[key[0]] else b): v for b, v in m.items()}
                         for key, m in self.ref.maps.items()}
        self.check(drain=False)


def build(c: Cluster, top):
    """Leaders elected, steady proposals that leave group g's leader g % SPREAD ids behind, a truncation (every floor > 0),
    then a step that neither delivers nor ticks: nothing is in flight afterwards.  Shifts both sides so that the highest
    block of any group is `top` (or, with top = None, so that the floors sit near 2^30 + 2^29 and the rows move by an
    odd count), and returns K."""
    G = c.G
    for api in c.apis:
        _bootstrap(api, G, c.R)
    c.launch("run", 10, 10, 0)
    c.call("leader_table")
    c.launch("run_tokens", 24, [[0 if k < g % SPREAD else (k << 32) + g + 1 for g in range(G)] for k in range(24)])
    c.call("truncate", 4)
    c.check(drain=False)
    with pytest.raises(Exception, match="E_INVAL"):
        c.ora.shift_ids(1 << 20)                    # mail in flight: refused
    for api in c.apis:
        api.step(c.now + DT, flags=0)               # the quiet tick
    c.now += DT
    c.check()
    st = [c.ora.query(g, 1) for g in range(G)]
    c.floor = [int(s.chain_floor) for s in st]
    assert min(c.floor) > 0
    hi = max(int(c.ora.query(g, n).max_key) for g in range(G) for n in range(1, c.R + 1))
    if top is None:
        K = (3 << 29) - min(c.floor)
        K += 1 - K % 2
    else:
        K = top - hi
    c.shift(K)
    return K


def _fold_ok(api, n_ticks, n_synth):
    """Groups sym_enter lets into the fold, by its room rule alone (every group is otherwise steady here)."""
    G, R = api.n_groups, api.n_replicas
    grow = n_ticks * (1 + n_synth) + 2
    st = api.query_many([(g, n) for g in range(G) for n in range(1, R + 1)])
    out = 0
    for g in range(G):
        rows = st[g * R:(g + 1) * R]
        lead = [x for x in rows if x.role == abi.ROLE_LEADER]
        if len(lead) != 1 or any(x.fault or not x.alive for x in rows):
            continue
        mk = lead[0].max_key
        out += mk + grow < LIMIT and mk + grow < lead[0].chain_floor + api.cfg.chain_capacity
    return out


def scenario(c: Cluster, base):
    top = {"a": None, "b": LIMIT - 80, "c": LIMIT - 43}[base]
    K = build(c, top)
    G, R = c.G, c.R
    floors = [int(c.ora.query(g, 1).chain_floor) for g in range(G)]
    if base == "a":
        assert K % 128 % 2 == 1 and min(floors) > (3 << 29) - 200
    else:
        assert all(f + c.ora.cfg.chain_capacity > LIMIT for f in floors)     # the window straddles 2^31
    # the fused calls, explicit and fused truncation, compaction
    c.launch("run_tokens", 4, [[0 if k == 2 else (77 << 40) + (k << 20) + g + 1 for g in range(G)] for k in range(4)])
    c.launch("run_token_runs", 4, 4, [(0 if g % 9 == 4 else (5 << 44) + g + 1, 1 << 32) for g in range(G)])
    c.call("truncate", 5)
    c.call("compact")
    c.check(drain=False)
    c.call("set_auto_truncate", 6)
    # steady appends: at base (c) sym_enter declines the groups whose next launch could reach 2^31, step_kernel runs them,
    # and each leader faults on the append of id 2^31 with its head at 2^31 - 1
    for k in range(12):
        want = _fold_ok(c.ora, 4, 1)
        c.launch("run", 4, 4, 1)
        if k >= 1:
            assert c.fold_counts[-1] == want, (k, c.fold_counts[-1], want)
    leaders = [s for s in c.ora.query_many([(g, n) for g in range(G) for n in range(1, R + 1)]) if s.role == abi.ROLE_LEADER]
    if base == "c":
        assert len(leaders) == G and min(c.fold_counts[-12:]) == 0 < c.fold_counts[-12]
        for s in leaders:
            assert (s.fault, s.head) == (abi.FAULT_ENGINE_CHAIN_CAPACITY, LIMIT - 1)
    else:
        assert all(s.fault == 0 and s.head < LIMIT for s in leaders)
    # leaders killed, every replica reopened from its exported chain: elections, and the new leaders' first append faults
    # (a restarted chain has id_gen == head, SURVEY N2)
    c.call("kill_leaders", 3, 500)
    c.call("set_auto_truncate", None)
    targets = [(g, n) for g in range(G) for n in range(1, R + 1)]
    chains = c.call("chain_export_many", targets)
    assert max(b[0] for _, _, bl in chains for b in bl) < LIMIT
    for api in c.apis:
        api.node_restart_many(c.now, [(g, n, bl, commit, ck) for (g, n), (commit, ck, bl) in zip(targets, chains)])
    for (g, n) in targets:
        c.ref.clear(g, n)
    c.check(drain=False)
    for k in range(4):
        c.launch("run", 10, 10, 1)
    faults = {s.fault for s in c.ora.query_many([(g, n) for g in range(G) for n in range(1, R + 1)])}
    if R == 3:                                      # (at R >= 5 the duplicated VoteRequests never elect, SURVEY N3)
        assert abi.FAULT_APPEND_ID_NOT_GT_HEAD in faults, faults
    return K


@pytest.mark.parametrize("base", ["a", "b", "c"])
@pytest.mark.parametrize("R", [3, 5, 7])
def test_shifted_ids_on_device_code(R, base, monkeypatch):
    scenario(Cluster(_emu, 33, R, monkeypatch), base)


@pytest.mark.gpu
@pytest.mark.parametrize("base", ["b", "c"])
def test_shifted_ids_4096x5_on_gpu(base, monkeypatch):
    scenario(Cluster(_gpu, 4096, 5, monkeypatch, sample=61), base)


# ---- ABI input at the limit ---------------------------------------------------------------------------------------------

def case_restart_at_the_limit(make, monkeypatch):
    """jr_node_restart(_many) refuses a block id, a next or a commit at 2^31 and leaves the engine untouched; a chain that
    reaches 2^31 - 1 at the top of a straddling window is taken, and equals the oracle.  Ids are below 2^31 (D4) wherever
    they appear in a persisted chain: a `next` names a parent, which is a block id too."""
    c = Cluster(make, 5, 3, monkeypatch)
    build(c, LIMIT - 80)
    g, n = 2, 3
    (commit, ck, blocks), = c.call("chain_export_many", [(g, n)])
    top, tok = blocks[-1][0], 99
    full = blocks + [(b, b - 1, tok + b) for b in range(top + 1, LIMIT)]          # up to 2^31 - 1
    floor = int(c.ora.query(g, n).chain_floor)
    assert floor + c.ora.cfg.chain_capacity > LIMIT and full[-1][0] == LIMIT - 1
    ok = dict(group=g, node=n, commit=LIMIT - 1, first_block=0, n_blocks=len(full), commit_key=1)
    bad = [
        ([ok], full[:-1] + [(LIMIT, LIMIT - 2, 1)]),                 # id 2^31 (still inside the window)
        ([ok], full[:-1] + [(LIMIT - 1, LIMIT, 1)]),                 # next 2^31
        ([ok], full[:-1] + [(LIMIT - 1, 0xFFFFFFFE, 1)]),            # next 2^32-2
        ([dict(ok, commit=LIMIT)], full),                            # commit 2^31
        ([dict(ok, commit=0xFFFFFFFE)], full),                       # commit 2^32-2
    ]
    for e in c.engs:
        before = e.save()
        for case in bad:
            assert _restart_raw(e, *case) == abi.E_INVAL, (e.kind, case[0], case[1][-1])
            assert e.save() == before, (e.kind, case[0], case[1][-1])
        with pytest.raises(Exception, match="E_INVAL"):             # the one-replica call: the same rule
            e.node_restart(g, n, c.now, full, LIMIT)
        assert e.save() == before
    for case in bad:
        chain, blk = case
        with pytest.raises(Exception, match="E_INVAL"):
            c.ora.node_restart(g, n, c.now, blk, chain[0]["commit"], True)
    for api in c.apis:
        api.node_restart_many(c.now, [(g, n, full, LIMIT - 1, True)])
    c.ref.clear(g, n)
    st = c.ora.query(g, n)
    assert (st.head, st.commit, st.id_gen, st.max_key) == (LIMIT - 1,) * 4
    c.check(drain=False)
    c.launch("run", 6, 6, 1)                                         # it follows the group's leader from there on


def _read_raw(api, first, count):
    g, n = (C.c_uint32 * 1)(0), (C.c_uint32 * 1)(1)
    f, k = (C.c_uint64 * 1)(first), (C.c_uint32 * 1)(count)
    out, present = (abi.Block * max(count, 1))(), (C.c_uint8 * max(count, 1))()
    st = api._fn("chain_read_many")(api._h, g, n, f, k, C.c_size_t(1), out, present)
    return st, [out[i].id for i in range(count)], [present[i] for i in range(count)]


def case_chain_read_at_the_limit(make):
    """jr_chain_read(_many): a range past 2^32 - 2 is refused, also when first_id + count wraps in u64; a range that ends
    at 2^32 - 1 answers with exactly the ids asked for, absent (no block is ever stored at or above 2^31)."""
    api = make(2, 3, chain_capacity=100)
    for first, count in ((1 << 64) - 1, 1), ((1 << 64) - 5, 10), (1 << 32, 1), \
                        ((1 << 32) - 1, 1), ((1 << 32) - 10, 10):
        assert _read_raw(api, first, count)[0] == abi.E_INVAL, (first, count)
        with pytest.raises(Exception, match="E_INVAL"):
            api.chain_read(0, 1, first, count)
    for first, count in ((1 << 32) - 11, 10), ((1 << 32) - 2, 1), (LIMIT - 3, 6), ((1 << 32) - 1, 0):
        st, ids, present = _read_raw(api, first, count)
        assert st == abi.OK and ids == list(range(first, first + count)) and not any(present), (first, count)


def test_restart_at_the_limit_on_device_code(monkeypatch):
    case_restart_at_the_limit(_emu, monkeypatch)


def test_chain_read_at_the_limit_on_device_code():
    case_chain_read_at_the_limit(_emu)


@pytest.mark.gpu
def test_restart_at_the_limit_on_gpu(monkeypatch):
    case_restart_at_the_limit(_gpu, monkeypatch)


@pytest.mark.gpu
def test_chain_read_at_the_limit_on_gpu():
    case_chain_read_at_the_limit(_gpu)


# ---- the headline shape -----------------------------------------------------------------------------------------------

REC = np.dtype([("group", "<u4"), ("hdr", "<u4"), ("id0", "<u4"), ("addr", "<u4"), ("tok0", "<u8"), ("stride", "<u8")])


def _records_np(api):
    ptr, batch = C.POINTER(abi.FsmRecord)(), abi.FsmBatch()
    assert api._lib.jr_fsm_records_async(api._h) == abi.OK
    assert api._lib.jr_fsm_records_wait(api._h, C.byref(ptr), C.byref(batch)) == abi.OK
    return np.frombuffer(C.string_at(ptr, batch.n_records * REC.itemsize), REC).copy()


def _warm_up_and_quiet(apis, G):
    for api in apis:
        _bootstrap(api, G, api.n_replicas)
        api.run(DT, DT, 10, 0)
        api.leader_table()
    toks = [[0 if k < g % SPREAD else (k << 32) + g + 1 for g in range(G)] for k in range(24)]
    for api in apis:
        api.run_tokens(11 * DT, DT, toks)
        api.truncate(4)
        api.discard_fsm()
        api.step(35 * DT, flags=0)                                   # the quiet tick
        api.discard_fsm()
    return 36 * DT


@pytest.mark.gpu
def test_shift_commutes_65536x5_on_gpu():
    """An engine at base 0 and one shifted to base K, driven alike at 65,536 x 5: every output of the second is the first's
    mapped through f.  No oracle is needed, so the headline shape is cheap."""
    G, R = 65536, 5
    cfg = dict(CFG, seed=3, fsm_host_records=G * R * 16, flags=CAP)
    a, b = _gpu(G, R, **cfg), _gpu(G, R, **cfg)
    b.cfg_dict = cfg
    now = _warm_up_and_quiet((a, b), G)
    floor = np.array([s.chain_floor for s in a.query_many([(g, 1) for g in range(G)])], np.int64)
    K = (3 << 29) - int(floor.min())
    K += 1 - K % 2
    shift_engine(b, K)

    def back(v, g):                                                  # f^-1 of group g's id v
        return v - K if v >= floor[g] + K else v

    sample = [(g, n) for g in range(0, G, 251) for n in range(1, R + 1)]
    id_fields = ("head", "commit", "id_gen", "max_key", "chain_floor")

    def same(launched=True):
        assert a.fold_count() == b.fold_count() and a.fault_count() == b.fault_count()
        la, lb = a.leader_table(), b.leader_table()
        assert la == [(t, l, back(c, g)) for g, (t, l, c) in enumerate(lb)]
        for (g, n), sa, sb in zip(sample, a.query_many(sample), b.query_many(sample)):
            da, db = sa.as_dict(), sb.as_dict()
            for k in id_fields:
                db[k] = back(db[k], g)
            db["progress_head"] = [back(v, g) for v in db["progress_head"]]
            assert da == db, (g, n)
        ra, rb = _records_np(a), _records_np(b)
        kind, count = rb["hdr"] & 3, rb["hdr"] >> 8
        lo = floor[rb["group"]] + K
        ids = (kind <= abi.FSMR_NOTIFY) & (rb["id0"] >= lo)
        rb["id0"][ids] -= np.uint32(K)
        nxt = (kind == abi.FSMR_APPLY) & (count == 1) & ((rb["stride"] & 0xFFFFFFFF).astype(np.int64) >= lo)
        rb["stride"][nxt] -= np.uint64(K)
        assert (len(ra) > G) == launched and np.array_equal(ra, rb)

    same(launched=False)
    for k in range(4):
        for api in (a, b):
            api.run(now, DT, 8, 1)
        now += 8 * DT
        same()
    toks = [[(9 << 40) + (k << 20) + g + 1 if (g + k) % 5 else 0 for g in range(G)] for k in range(8)]
    for api in (a, b):
        api.run_tokens(now, DT, toks)
        api.truncate(5)
        api.compact()
    now += 8 * DT
    same()


@pytest.mark.gpu
def test_crossing_2_31_65536x5_on_gpu():
    """Base (c) at 65,536 x 5 against the oracle through the digests: sym_enter declines exactly the groups whose launch
    could reach 2^31, and every leader faults on the append of 2^31 with its head at 2^31 - 1, as the oracle's do."""
    G, R = 65536, 5
    cfg = dict(CFG, seed=4, fsm_host_records=G * R * 16)
    eng = _gpu(G, R, flags=CAP, **cfg)
    ora = _oracle(G, R, flags=CAP, n_threads=16, **cfg)
    eng.cfg_dict = dict(cfg, flags=CAP)
    now = _warm_up_and_quiet((eng, ora), G)
    top = max(s.max_key for s in ora.query_many([(g, 1) for g in range(G)]))
    K = LIMIT - 40 - top
    shift_engine(eng, K)
    ora.shift_ids(K)
    assert eng.state_digest() == ora.state_digest()
    for api in (eng, ora):
        api.set_auto_truncate(6)
    folds = []
    for k in range(13):
        want = _fold_ok(eng, 4, 1)
        for api in (eng, ora):
            api.run(now, DT, 4, 1)
            api.discard_fsm()
        now += 4 * DT
        folds.append(eng.fold_count())
        if k:
            assert folds[-1] == want, (k, folds, want)
        assert eng.state_digest() == ora.state_digest(), k
        assert eng.leader_table() == ora.leader_table() and eng.fault_count() == ora.fault_count(), k
    assert folds[1] == G and folds[-1] == 0
    lead = [s for s in eng.query_many([(g, 1) for g in range(G)])]
    assert all((s.role, s.fault, s.head) == (abi.ROLE_LEADER, abi.FAULT_ENGINE_CHAIN_CAPACITY, LIMIT - 1) for s in lead)
