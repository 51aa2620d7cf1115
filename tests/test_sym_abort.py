"""The fold's mid-launch fallback (josefine_b200/csrc/sym_fold.cuh, DESIGN.md §3b): a lane of sym2_kernel that meets
anything outside the canonical evolution aborts, the group is handed back to step_kernel, and the abort must cost time,
never correctness.  Here the aborts are constructed -- at a chosen tick, on a chosen lane, at chosen positions in the
CTAs of sym2_kernel and step_kernel -- and after every launch the folding engine must equal the never-folding engine
and the oracle on everything: the Instruction stream, replica states, leader tables, the whole block-table window of
every replica around the aborted groups (ids above every head included), and the checkpoint bytes segment by segment
(the only place the outboxes, the progress planes and the queues are compared exactly).

The host build of the device code (tests/emu) is built with JR_SYM_ABORT_LOG: it records, per group and lane, the
first abort site and its tick (jr_sym_abort_read), so every test also checks that the abort it constructed is the one
that fired, and that no other did."""
import ctypes as C
import struct

import numpy as np
import pytest

from josefine_b200 import abi
from josefine_b200.raft import RaftError
from tests import parity
from tests.stream_cases import _bootstrap
from tests.test_sym_fold import CAP, _emu, _gpu, _oracle, same

# abort sites (SA_* in sym_fold.cuh) and lanes (0 = the leader's side, 1 = the followers')
SA_FETCH_F, SA_FIFO_L, SA_FIFO_F, SA_COMMIT, SA_CLIENT, SA_HBR, SA_EXTEND, SA_PROPOSAL = range(1, 9)
LEAD, FOLLOW = 0, 1
ABSENT = 0xFFFFFFFF
GROUPS_PER_CTA = 32                 # step_kernel's group block (engine.cu)
SYM2_GROUPS = 64                    # groups per sym2_kernel CTA (sym_fold.cuh)


def trio(make, G, R, **cfg):
    cfg.setdefault("flags", CAP)
    fold = make(G, R, **cfg)
    plain = make(G, R, **dict(cfg, flags=cfg["flags"] | abi.F_NO_SYMMETRIC_FOLD))
    return fold, plain, _oracle(G, R, **cfg)


def aborts_of(api):
    """The abort log of the host build; None on the GPU build (which has no log)."""
    return api.sym_aborts() if hasattr(api, "sym_aborts") else None


# ---- checkpoint bytes ------------------------------------------------------------------------------------------------
# jr_engine_save writes a SaveHeader {magic, bytes, jr_config, cur, route_valid, step_index} and then the segments of
# save_segments (engine.cu), in this order.

def _segments(api):
    cfg, G, R = api.cfg, api.n_groups, api.n_replicas
    Gp = (G + GROUPS_PER_CTA - 1) // GROUPS_PER_CTA * GROUPS_PER_CTA
    plane = R * Gp
    rows = 1
    while rows < cfg.chain_capacity:
        rows <<= 1
    U, F = cfg.mailbox_units, cfg.fsm_units
    seg = [("p0", plane * 16), ("p1", plane * 16), ("p2", plane * 16), ("p3", plane * 16),
           ("pr", plane * ((R + 3) // 4) * 16), ("mk", plane * 4), ("qt", plane * 4 * 16), ("dg", plane * 16),
           ("cn", plane * 8), ("cnext", plane * rows * 4), ("ctok", plane * rows * 8),
           ("ob0", plane * U * 16), ("ob1", plane * U * 16), ("oc0", plane * 4), ("oc1", plane * 4),
           ("fs", plane * ((2 * F) if cfg.flags & abi.F_CAPTURE_FSM else 1) * 16), ("fc", plane * 8),
           ("tb", Gp * 4), ("route", G * 4)]
    if cfg.flags & abi.F_CLIENT_RESPONSES:
        seg.append(("pn", (2 * abi.NOTIFY_RUNS * plane + (plane + 3) // 4 + plane) * 16))
    return seg, Gp, plane, rows


def checkpoint(api):
    blob = api.save()
    hdr = 16 + C.sizeof(abi.Config) + 16
    seg, Gp, plane, rows = _segments(api)
    assert len(blob) == hdr + sum(n for _, n in seg), "checkpoint layout changed: update _segments"
    cur = struct.unpack_from("<I", blob, 16 + C.sizeof(abi.Config))[0]
    out, at = {"cur": cur}, hdr
    for name, n in seg:
        out[name] = np.frombuffer(blob, dtype=np.uint8, count=n, offset=at)
        at += n
    return out


def same_checkpoint(a, b):
    """The folding engine's checkpoint equals the never-folding engine's, segment by segment.  Masked are only bytes no
    reader can observe before they are overwritten (each mask names the code that does it); FS / FC are compared through
    the drain instead (same()), because folded followers legitimately share one set of APPLY records."""
    ca, cb = checkpoint(a), checkpoint(b)
    G, R, U = a.n_groups, a.n_replicas, a.cfg.mailbox_units
    _, Gp, plane, rows = _segments(a)
    assert ca["cur"] == cb["cur"]
    live = 1 - ca["cur"]        # the outbox the last tick wrote; the next launch reads it (prv = 1 - cur)
    for name in ca:
        if name in ("cur", "fs", "fc"):
            continue
        x, y = ca[name], cb[name]
        if name == "ctok":
            # the token of an absent row: every reader of ctok looks at the row's cnext first and ignores the token of
            # an ABSENT one (fetch / fetch_sent callers, sym_enter's compare, step_kernel's table reads, chain_read)
            absent = ca["cnext"].view(np.uint32) == ABSENT
            assert (absent == (cb["cnext"].view(np.uint32) == ABSENT)).all()
            x = np.where(absent, 0, x.view(np.uint64))
            y = np.where(absent, 0, y.view(np.uint64))
        elif name in ("ob0", "ob1", "oc0", "oc1"):
            b = int(name[2])
            if b != live:
                # the outbox of the launch's second-to-last tick (step_kernel) or an older one (the fold writes only
                # the last tick's): the next launch's first tick resets it (PH_RESET_OUT) and fills it before any read
                continue
            if name.startswith("ob"):
                # units at or beyond a mailbox's count: every reader (step_kernel's delivery, sym_enter) stops at oc,
                # and the sender writes a unit before it raises oc over it
                oc = ca["oc%d" % b].view(np.uint32).reshape(R, Gp)
                k = np.arange(U).reshape(U, 1, 1)
                used = k < oc.reshape(1, R, Gp)
                x = np.where(used, x.view(np.uint32).reshape(U, R, Gp, 4).transpose(3, 0, 1, 2), 0)
                y = np.where(used, y.view(np.uint32).reshape(U, R, Gp, 4).transpose(3, 0, 1, 2), 0)
        elif name == "pn":
            # the fsm::Driver maps: [2 * run + half][replica][group] units, then the run counts, then the restart marks.
            # Runs at or beyond a replica's count: fsm_respond_kernel reads runs [0, count) only and writes a run before
            # it raises the count over it (jr_engine_reset zeroes the counts, not the runs)
            nr = 2 * abi.NOTIFY_RUNS * plane * 4
            cnt = x.view(np.uint32)[nr:nr + plane]
            assert np.array_equal(cnt, y.view(np.uint32)[nr:nr + plane]), "fsm::Driver run counts differ"
            used = (np.arange(abi.NOTIFY_RUNS).reshape(-1, 1, 1) < cnt.reshape(1, 1, plane))
            used = np.broadcast_to(used, (abi.NOTIFY_RUNS, 2, plane)).reshape(-1, 1)
            runs = lambda v: np.where(used, v.view(np.uint32)[:nr].reshape(-1, 4), 0)
            x = np.concatenate([runs(x).reshape(-1), x.view(np.uint32)[nr:]])
            y = np.concatenate([runs(y).reshape(-1), y.view(np.uint32)[nr:]])
        if not np.array_equal(x, y):
            xs, ys = np.asarray(x).reshape(-1), np.asarray(y).reshape(-1)
            i = int(np.flatnonzero(xs != ys)[0])
            raise AssertionError(f"checkpoint segment {name} differs at element {i} of {xs.size}: {xs[i]} vs {ys[i]}")


def same_windows(apis, groups):
    """Every replica of `groups` over its whole window [floor, floor + chain_capacity), id for id, ids above every head
    included: a row an aborted lane wrote and step_kernel did not rewrite would sit there."""
    a = apis[0]
    cap = a.cfg.chain_capacity
    reqs = [(g, n, max(int(a.query(g, n).chain_floor), 0), cap) for g in sorted(groups) for n in range(1, a.n_replicas + 1)]
    want = apis[0].chain_read_many(reqs)
    for other in apis[1:]:
        got = other.chain_read_many(reqs)
        for r, x, y in zip(reqs, want, got):
            assert x == y, f"window of group {r[0]} node {r[1]} from id {r[2]} differs"


def neighbours(groups, G):
    """The aborted groups and the other groups of their step_kernel blocks."""
    return {h for g in groups for h in range(g // GROUPS_PER_CTA * GROUPS_PER_CTA, min(G, (g // GROUPS_PER_CTA + 1) * GROUPS_PER_CTA))}


def check_launch(apis, aborted, refused=(), log=None):
    """After a launch: the fold count, the abort log, the windows around the aborts, the checkpoint bytes, then same()."""
    fold, plain = apis[0], apis[1]
    G = fold.n_groups
    assert fold.fold_count() == G - len(refused) - len(aborted), (fold.fold_count(), sorted(aborted), sorted(refused))
    assert plain.fold_count() == 0
    got = aborts_of(fold)
    if got is not None and log is not None:
        assert got == log, f"abort log {sorted(got.items())} != expected {sorted(log.items())}"
    same_windows(apis, neighbours(set(aborted) | set(refused), G) or {0, G - 1})
    same_checkpoint(fold, plain)
    same(apis, chain_ids=0)


# ---- where the aborting groups sit ------------------------------------------------------------------------------------

def positions(G, every=1):
    """Groups at the edges that matter: the first and last group of a sym2_kernel CTA (both warp pairs; even and odd
    CTAs, whose leader lanes sit in different warps), the first and last group of a step_kernel block whose other groups
    fold, and the tail CTA when G is not a multiple of 64.  every > 1: only CTAs 0, 1 and every `every`-th pair after
    them, and the last two."""
    out = []
    n_ctas = (G + SYM2_GROUPS - 1) // SYM2_GROUPS
    for c in range(n_ctas):
        if every > 1 and c > 1 and c < n_ctas - 2 and (c // 2) % every:
            continue
        base = c * SYM2_GROUPS
        for gi in (0, 31, 32, SYM2_GROUPS - 1):
            if base + gi < G:
                out.append(base + gi)
        if base + SYM2_GROUPS > G:
            out.append(G - 1)
    return sorted(set(out))


def tick_choices(n):
    return [0, 1, n // 2, n - 2, n - 1]


# ---- 1. the leader lane: a proposal for a follower at a chosen tick ----------------------------------------------------

def case_proposal_aborts(make, G, R, lead=1, n=9, rounds=2, every=1, cfg_over=None, auto_truncate=None):
    """Dense jr_run_proposals: every group proposes to its leader at every tick, except that group g of `groups` proposes
    to a follower at its tick t_g -- a proxied ClientRequest, which the fold does not model: the leader lane aborts at
    exactly t_g.  Each round moves every group to another of the ticks 0, 1, n/2, n-2, n-1; a canonical launch follows,
    in which every group folds again (those whose proxied request is still in flight after an abort at the last tick
    are refused at entry first, and fold one launch later)."""
    cfg = dict(seed=17 + R, chain_capacity=128, fsm_units=64, fsm_host_records=G * R * 64, mailbox_units=64)
    cfg.update(cfg_over or {})
    apis = trio(make, G, R, **cfg)
    groups = positions(G, every)
    follower = 1 if lead != 1 else R
    tok = [1 << 36]

    def props(ticks, aborts):
        rows = []
        for t in range(ticks):
            row = []
            for g in range(G):
                tok[0] += 1
                row.append((follower if aborts.get(g) == t else lead, tok[0] * 4096 + g))
            rows.append(row)
        return rows

    for api in apis:
        _bootstrap(api, G, R, node=lead)
        api.run(100, 100, 12, 1)
        api.leader_table()
        if auto_truncate is not None:
            api.set_auto_truncate(auto_truncate)
    now = 1300
    p = props(n, {})
    for api in apis:
        api.run_proposals(now, 100, p)
    now += 100 * n
    check_launch(apis, aborted=[], log={})
    choices = tick_choices(n)
    for rnd in range(rounds):
        aborts = {g: choices[(i + rnd) % len(choices)] for i, g in enumerate(groups)}
        p = props(n, aborts)
        for api in apis:
            api.run_proposals(now, 100, p)
        now += 100 * n
        check_launch(apis, aborted=aborts, log={(g, LEAD): (SA_PROPOSAL, t) for g, t in aborts.items()})
        late = [g for g, t in aborts.items() if t == n - 1]      # their proxied request reaches the leader next launch
        for refused in (late, []):
            p = props(n, {})
            for api in apis:
                api.run_proposals(now, 100, p)
            now += 100 * n
            check_launch(apis, aborted=[], refused=refused, log={})
            if not late:
                break
    return apis


@pytest.mark.parametrize("R,lead", [(2, 1), (3, 2), (5, 1), (5, 4), (8, 3)])
def test_proposal_aborts_on_device_code(R, lead):
    case_proposal_aborts(_emu, 150 if R <= 5 else 72, R, lead=lead)


def test_proposal_aborts_split_launches_on_device_code(monkeypatch):
    """JR_PARTS=3: step_kernel re-runs the aborted groups in split launches, next to folded groups of the same block."""
    monkeypatch.setenv("JR_PARTS", "3")
    case_proposal_aborts(_emu, 150, 3, n=12)


def test_proposal_aborts_auto_truncate_on_device_code():
    """jr_set_auto_truncate: the fused truncation of sym2_kernel must skip the aborted groups; truncate_kernel takes
    them.  (A small window, so that the floors really move.)"""
    apis = case_proposal_aborts(_emu, 150, 5, lead=3, rounds=3, auto_truncate=4, cfg_over=dict(chain_capacity=64))
    assert min(int(apis[0].query(g, 1).chain_floor) for g in range(150)) > 20


# ---- 2. the leader lane: its raw Instruction FIFO fills at a chosen tick -----------------------------------------------

def same_lossy(apis):
    """After a launch whose Instructions did not all fit the raw FIFO (step_kernel drops the excess and counts it): both
    engines report the same loss, the same ClientResponse runs (JR_F_CLIENT_RESPONSES), the same fsm::Driver maps (in
    the checkpoint), and the states, leader tables and fault counts of the oracle, whose stream has no such bound."""
    fold, plain, ora = apis
    got = []
    for api in (fold, plain):
        with pytest.raises(RaftError) as err:
            api.fsm_records()
        resp = None
        if api.cfg.flags & abi.F_CLIENT_RESPONSES:
            recs, batch = api.fsm_responses()
            resp = ([tuple(bytes(r)) for r in recs], batch.n_records, batch.n_dropped)
        got.append((str(err.value), resp))
    assert got[0] == got[1]
    assert "dropped" in got[0][0]
    ora.discard_fsm(strict=False)
    same_checkpoint(fold, plain)
    for other in (plain, ora):
        parity.compare_states(fold, other)
        assert fold.state_digest() == other.state_digest()
        assert fold.leader_table() == other.leader_table()
        assert fold.fault_count() == other.fault_count()


# fsm_raw_units = 32 (the smallest jr_engine_create takes): jr_run cuts a call into launches of at most 10 ticks.  The
# leader emits n_synth Notify per tick and, once the commit follows them, as many APPLY, so from a steady start its FIFO
# fills at tick 6 with 3 proposals per tick and at tick 5 with 4: the last tick of 7, the middle of 10, n - 2 of 7.
@pytest.mark.parametrize("n_synth,n,tick", [(3, 7, 6), (3, 10, 6), (4, 7, 5)])
@pytest.mark.parametrize("responses", [False, True])
def test_leader_fifo_aborts_on_device_code(n_synth, n, tick, responses):
    G, R = 70, 3
    flags = CAP | (abi.F_CLIENT_RESPONSES if responses else 0)
    apis = trio(_emu, G, R, seed=5, chain_capacity=256, fsm_units=256, fsm_host_records=G * R * 64, fsm_raw_units=32, flags=flags)
    for api in apis:
        _bootstrap(api, G, R, node=2)
        api.run(100, 100, 10, 1)
        api.leader_table()
    now = 1100
    for rnd in range(2):
        for api in apis:
            api.run(now, 100, 10, 1)                 # canonical: every group folds
        now += 1000
        check_launch(apis, aborted=[], log={})
        for api in apis:
            api.run(now, 100, n, n_synth)
        now += 100 * n
        assert apis[0].fold_count() == 0
        assert aborts_of(apis[0]) == {(g, LEAD): (SA_FIFO_L, tick) for g in range(G)}
        same_windows(apis, range(G))
        same_lossy(apis)


@pytest.mark.gpu
@pytest.mark.parametrize("G,R,lead,every", [(8257, 5, 1, 4), (2100, 8, 2, 2)])
def test_proposal_aborts_on_gpu(G, R, lead, every):
    """sym2_kernel on the H100: aborts at every position kind and tick, spread over the grid, with a tail CTA (8,257 =
    129 CTAs of 64 + 1), and R = 8."""
    case_proposal_aborts(_gpu, G, R, lead=lead, rounds=1, every=every)


@pytest.mark.gpu
def test_proposal_aborts_auto_truncate_on_gpu():
    apis = case_proposal_aborts(_gpu, 8257, 5, lead=2, rounds=2, every=8, auto_truncate=4, cfg_over=dict(chain_capacity=64))
    assert min(int(apis[0].query(g, 1).chain_floor) for g in range(0, 8257, 97)) > 20
