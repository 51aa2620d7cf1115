"""Client responses from the batched drain (JR_F_CLIENT_RESPONSES, jr_fsm_responses): fsm::Driver's notification map
(fsm.rs:57-81) run on the device over the Instructions that leave the engine.  Every case runs on the device code built
for the host and on the GPU, on folding and on never-folding (JR_F_NO_SYMMETRIC_FOLD) engines, and compares the expanded
responses per replica with a restatement of the Driver fed by the C++ oracle's drained Instructions -- and, where the
size allows, with BatchedDriver fed the same Instructions."""
import ctypes as C
import random

import numpy as np
import pytest

from josefine_b200 import abi, Address, BatchedDriver, Command, expand_responses
from tests.stream_cases import strided_tokens

CAP = abi.F_CAPTURE_FSM
RESP = abi.F_CLIENT_RESPONSES


def _oracle(g, r, **kw):
    from oracle.restated import RestatedCluster
    return RestatedCluster.create(g, r, **kw)


def _emu(g, r, **kw):
    from tests.emu.emu import EmuEngine
    return EmuEngine.create(g, r, **kw)


def _gpu(g, r, **kw):
    from josefine_b200 import RaftEngine
    return RaftEngine.create(g, r, **kw)


class DriverRef:
    """fsm.rs:57-81 per (group, node), fed Instructions in emission order: Notify inserts block_id -> (address, id)
    (fsm.rs:78-81, overwriting), Apply of a block other than 0 (fsm.rs:61-63) removes block.id and answers a hit
    (fsm.rs:66-76).  The map is unbounded, as in the reference."""

    def __init__(self):
        self.maps = {}

    def feed(self, instructions):
        out = []
        for ins in instructions:
            m = self.maps.setdefault((ins.group, ins.node), {})
            if ins.kind == abi.FSM_NOTIFY:
                m[ins.block.id] = (Address(ins.client_kind, ins.client_id), ins.block.data)
            elif ins.block.id != 0 and ins.block.id in m:
                to, tok = m.pop(ins.block.id)
                out.append((ins.group, ins.node, to, tok, ins.block.id))
        return sorted(out, key=lambda x: (x[0], x[1]))     # stable: apply order per replica

    def clear(self, group=None, node=None):
        if group is None:
            self.maps.clear()
        else:
            self.maps.pop((group, node), None)


class Pair:
    """An engine with JR_F_CLIENT_RESPONSES, the oracle, and the Driver restatement over the oracle's Instructions."""

    def __init__(self, make, G, R, fold=True, check_batched_driver=True, **cfg):
        flags = cfg.pop("flags", CAP)
        self.eng = make(G, R, flags=flags | RESP | (0 if fold else abi.F_NO_SYMMETRIC_FOLD), **cfg)
        self.ora = _oracle(G, R, flags=flags, **cfg)
        self.G, self.R = G, R
        self.ref = DriverRef()
        self.drv = BatchedDriver(lambda g, n: _Null(), {}) if check_batched_driver else None
        self.fsm_cap = max(1 << 16, G * R * 400)

    def both(self, name, *a, **kw):
        return [getattr(api, name)(*a, **kw) for api in (self.eng, self.ora)]

    def _expect(self, instructions):
        want = self.ref.feed(instructions)
        if self.drv is not None:
            rb = self.drv.feed(instructions)
            key = lambda g, n, to, tok: (g, n, to.kind, to.id, tok)   # noqa: E731
            assert sorted(key(r.group, r.node, r.to, r.request) for r in rb) == sorted(key(*w[:4]) for w in want)
        return want

    def responses(self):
        runs, batch = self.eng.fsm_responses()
        got = expand_responses(runs)
        assert batch.n_instructions == len(got) and batch.n_records == len(runs)
        return got, runs, batch

    def step(self, now, **kw):
        """jr_step with out_fsm: the step's drain answers what the oracle's step hands out."""
        re, ro = self.both("step", now, cap_fsm=self.fsm_cap, **kw)
        want = self._expect(ro.fsm)
        got, runs, batch = self.responses()
        assert got == want
        return got, re

    def drain(self, how="drain", strict=True):
        ins = self.ora.drain_fsm(cap=self.fsm_cap)
        if how == "drain":
            self.eng.drain_fsm(cap=self.fsm_cap)
        elif how == "discard":
            self.eng.discard_fsm(strict=strict)
        else:
            self.eng.fsm_records()
        want = self._expect(ins)
        got, runs, batch = self.responses()
        if strict:
            assert batch.n_dropped == 0
            assert got == want, f"engine {got[:6]}... != reference {want[:6]}..."
        return got, want, runs, batch

    def bootstrap(self, node=1):
        q = 0 if self.R == 1 else self.R // 2 + 1
        inj = []
        for g in range(self.G):
            inj.append(Command.timeout(g, node))
            inj += [Command.vote_response(g, node, 1, v, True) for v in range(1, self.R + 1) if v != node][:max(q - 1, 0)]
        self.step(0, flags=0, inject=inj)
        self.both("run", 100, 100, 10, 0)
        self.both("leader_table")
        self.drain()


class _Null:
    def transition(self, data):
        return data


MAKERS = {"emu": _emu, "gpu": _gpu}
FOLDS = [True, False]


def _params(where):
    marks = [pytest.mark.gpu] if where == "gpu" else []
    return [pytest.param(MAKERS[where], fold, id=f"{where}-{'fold' if fold else 'nofold'}", marks=marks) for fold in FOLDS]


ALL = _params("emu") + _params("gpu")


# ---- 1. known answers --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("make,fold", ALL)
def test_single_node_propose_is_answered_to_client(make, fold):
    """fsm_cases.case_single_node_propose_completes on the device path: leader.rs:177-194 Notify, commit, fsm.rs:66-76."""
    p = Pair(make, 1, 1, fold=fold)
    p.step(0, flags=0, inject=[Command.timeout(0, 1)])
    got, _ = p.step(0, flags=0, inject=[Command.client_request(0, 1, token=123)])
    assert got == [(0, 1, Address.client(), 123, 1)]


@pytest.mark.parametrize("make,fold", ALL)
def test_proxied_request_is_answered_to_the_follower(make, fold):
    """follower.rs:258-269 proxies with address Peer(follower); the leader's Driver answers Peer(2) (fsm.rs:67-76); the host
    relays Command.client_response (follower.rs:271-282)."""
    p = Pair(make, 1, 3, fold=fold)
    p.step(0, flags=0, inject=[Command.timeout(0, 1), Command.vote_response(0, 1, 1, 2, True)])
    p.step(100)
    p.step(200, inject=[Command.client_request(0, 2, token=77)])
    answered, relay = [], []
    for k in range(3, 12):
        got, res = p.step(100 * k, inject=relay)
        relay = [Command.client_response(g, to.id, tok) for g, node, to, tok, _ in got if to.kind == abi.ADDR_PEER]
        answered += got
    assert [(n, to, tok) for _, n, to, tok, _ in answered] == [(1, Address.peer(2), 77)]


@pytest.mark.parametrize("make,fold", ALL)
def test_notify_and_apply_in_one_batch_and_across_batches(make, fold):
    G, R = 8, 3
    p = Pair(make, G, R, fold=fold, chain_capacity=256, fsm_units=64)
    p.bootstrap()
    p.both("run_tokens", 1100, 100, [[1000 + g for g in range(G)]])
    got, *_ = p.drain()                                   # Notify only: pending across the drain
    assert got == []
    p.both("run", 1200, 100, 4, 0)
    got, *_ = p.drain()
    assert sorted((g, tok) for g, _, _, tok, _ in got) == [(g, 1000 + g) for g in range(G)]
    p.both("run_tokens", 1600, 100, [[2000 + g for g in range(G)]])
    p.both("run", 1700, 100, 4, 0)
    got, *_ = p.drain()                                   # Notify and Apply in the same batch
    assert sorted((g, tok) for g, _, _, tok, _ in got) == [(g, 2000 + g) for g in range(G)]


# ---- 2. steady state ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("R", [2, 3, 5, 7])
@pytest.mark.parametrize("make,fold", ALL)
def test_steady_token_runs(make, fold, R):
    G, S = 24, 33
    p = Pair(make, G, R, fold=fold, seed=R, chain_capacity=512, fsm_units=128)
    p.bootstrap()
    now = 1100
    total = 0
    for launch in range(5):
        p.both("run_token_runs", now, 100, S, [((launch + 1) << 40 | (g + 1) << 20, 1 << 8) for g in range(G)])
        now += 100 * S
        got, want, runs, batch = p.drain()
        total += len(got)
        per = {}
        for rc in runs:
            per[(rc.group, rc.node)] = per.get((rc.group, rc.node), 0) + 1
        assert max(per.values(), default=0) <= 2, "constant-stride tokens: at most 2 response runs per leader per launch"
    assert total >= G * (5 * S - 8)


# ---- 3. arbitrary tokens ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("make,fold", ALL)
def test_arbitrary_tokens_holes_and_misrouted(make, fold):
    G, R = 16, 5
    rng = random.Random(7)
    p = Pair(make, G, R, fold=fold, seed=4, chain_capacity=512, fsm_units=256)
    p.bootstrap()
    now = 1100
    for rnd in range(4):
        toks = [[rng.getrandbits(63) | 1 if rng.random() < 0.8 else 0 for _ in range(G)] for _ in range(12)]
        p.both("run_tokens", now, 100, toks)
        now += 1200
        props = [[(rng.choice([1, 1, 2, 3, 0]), rng.getrandbits(62) | 1) for _ in range(G)] for _ in range(6)]
        p.both("run_proposals", now, 100, props)     # proposals at followers: proxied to the leader (Peer(n))
        now += 600
        got, want, runs, _ = p.drain(how=["drain", "records"][rnd % 2])
        assert len(runs) <= len(got)
    p.both("run", now, 100, 10, 0)
    p.drain()


# ---- 5. lifecycle -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("make,fold", ALL)
def test_restart_reset_and_checkpoint(make, fold):
    G, R = 6, 3
    p = Pair(make, G, R, fold=fold, seed=2, chain_capacity=256, fsm_units=64)
    p.bootstrap()
    for api in (p.eng, p.ora):                      # followers silenced: notifications stay pending
        for g in range(G):
            for n in range(2, R + 1):
                api.set_alive(g, n, False)
    p.both("run_tokens", 1100, 100, strided_tokens(3, G, 0))
    p.drain()
    # node restart clears the replica's map (server.rs:80-81, fsm.rs:48): group 0 via restart, group 1 via restart_many
    for api in (p.eng, p.ora):
        exp = api.chain_export_many([(0, 1), (1, 1)])
        api.node_restart(0, 1, 1400, exp[0][2], exp[0][0], exp[0][1])
        api.node_restart_many(1400, [(1, 1, exp[1][2], exp[1][0], exp[1][1])])
    p.ref.clear(0, 1)
    p.ref.clear(1, 1)
    blob = p.eng.save()

    def revive_and_run(apis):
        for api in apis:
            for g in range(G):
                for n in range(2, R + 1):
                    api.set_alive(g, n, True)
            api.run(1500, 100, 12, 0)

    revive_and_run([p.eng, p.ora])
    first = p.drain()[0]
    assert first and {g for g, *_ in first} <= set(range(2, G))
    # restore -> the same run -> the same responses, response for response (the oracle keeps no checkpoints)
    p.eng.restore(blob)
    revive_and_run([p.eng])
    p.eng.drain_fsm(cap=p.fsm_cap)
    assert p.responses()[0] == first
    # jr_engine_reset clears every map (and forgets the last batch)
    from josefine_b200 import RaftError
    p.eng.restore(blob)
    assert p.eng._lib.jr_engine_reset(p.eng._h) == 0
    with pytest.raises(RaftError):
        p.eng.fsm_responses()
    p2 = Pair(make, G, R, fold=fold, seed=2, chain_capacity=256, fsm_units=64)
    p2.eng, p.eng = p.eng, None                          # the reset engine against a fresh oracle
    p2.bootstrap()
    p2.both("run_tokens", 1100, 100, strided_tokens(3, G, 0))
    p2.both("run", 1400, 100, 6, 0)
    assert p2.drain()[0]


@pytest.mark.parametrize("make,fold", ALL)
def test_restart_with_undrained_notifies_starts_a_new_map(make, fold):
    """A leader's Notifies are still undrained when it restarts (server.rs:80-81: the old process's Driver and its map die,
    fsm.rs:48: the new one starts empty).  The drain after the restart still carries them, but they belong to the old
    map: a new leader's block with the same id, applied by the restarted replica, must not answer the old client.  The
    reference is fed the oracle's pre-restart Instructions, then cleared, then fed the rest."""
    G, R = 16, 3
    p = Pair(make, G, R, fold=fold, seed=11, chain_capacity=256, fsm_units=64)
    p.bootstrap()
    for api in (p.eng, p.ora):
        for g in range(G):
            for n in (2, 3):
                api.set_alive(g, n, False)
    old = [[5000 + 100 * k + g for g in range(G)] for k in range(3)]
    p.both("run_tokens", 1100, 100, old)                  # block ids X.. appended at node 1, never committed
    p.ref.feed(p.ora.drain_fsm(cap=p.fsm_cap))           # the oracle's pre-restart stream; the engine keeps its own undrained
    for api in (p.eng, p.ora):                            # nodes 1 and 2 restart from what they committed
        exp = api.chain_export_many([(g, n) for g in range(G) for n in (1, 2)])
        chains = []
        for (g, n), (commit, ck, blocks) in zip([(g, n) for g in range(G) for n in (1, 2)], exp):
            chains.append((g, n, [b for b in blocks if b[0] <= commit], commit, ck))
        api.node_restart_many(1400, chains)
        for g in range(G):
            for n in (2, 3):
                api.set_alive(g, n, True)
    for g in range(G):
        p.ref.clear(g, 1)
        p.ref.clear(g, 2)
    p.both("run", 1400, 100, 20, 0)
    leaders = p.both("leader_table")[0]
    p.both("run_tokens", 3400, 100, [[9000 + 100 * k + g for g in range(G)] for k in range(3)])
    p.both("run", 3700, 100, 10, 0)
    got, want, _, _ = p.drain()
    assert not [x for x in got if x[3] < 9000], "an old client was answered"
    assert {lid for _, lid, _ in leaders} >= {1, 2}, "some groups must elect node 2: node 1 then applies its block X"
    assert len(got) >= 2 * G
    # a restart followed by jr_step: the step drops the undrained Instructions (PH_RESET_FSM), the map starts empty
    p.both("run_tokens", 4700, 100, [[12000 + g for g in range(G)]])
    for api in (p.eng, p.ora):
        api.node_restart_many(4800, [(g, 3, None, 0, None) for g in range(G)] if api is p.eng else
                              [(g, 3, *_committed(api, g, 3)) for g in range(G)])
    for g in range(G):
        p.ref.clear(g, 3)
    p.step(4800)


def _committed(api, g, n):
    commit, ck, blocks = api.chain_export_many([(g, n)])[0]
    return blocks, commit, ck


def _save_layout(cfg, G, R):
    """Byte offsets of the FS and FC segments in a jr_engine_save checkpoint (engine.cu save_segments, in order)."""
    Gp = (G + 31) // 32 * 32
    plane = R * Gp
    rows = 1
    while rows < cfg["chain_capacity"]:
        rows <<= 1
    at = 104                                              # SaveHeader
    sizes = [plane * 16] * 4 + [plane * ((R + 3) // 4) * 16, plane * 4, plane * 4 * 16, plane * 16, plane * 8,
                                plane * rows * 4, plane * rows * 8, plane * cfg["mailbox_units"] * 16,
                                plane * cfg["mailbox_units"] * 16, plane * 4, plane * 4]
    at += sum(sizes)
    return at, at + plane * 2 * cfg["fsm_units"] * 16, plane


@pytest.mark.parametrize("make", [pytest.param(_emu, id="emu"), pytest.param(_gpu, id="gpu", marks=pytest.mark.gpu)])
def test_overwrite_and_split_of_pending_runs(make):
    """The map's rarer paths on one hand-made stream, loaded through a checkpoint: Notify 5..8 (one run), Apply 7 (the run
    splits), Notify 6 again (HashMap insert overwrites, fsm.rs:80), Apply 6, 8, 5 and the genesis block 0 (skipped,
    fsm.rs:61-63).  The expected answers come from the Driver restatement over jr_fsm_expand of the same records."""
    import struct
    from josefine_b200.raft import expand_records
    cfg = dict(chain_capacity=64, mailbox_units=64, fsm_units=16)
    eng = make(1, 1, flags=CAP | RESP, **cfg)
    blob = bytearray(eng.save())
    fs_at, fc_at, plane = _save_layout(cfg, 1, 1)
    client = abi.ADDR_CLIENT << 16
    recs = [(abi.FSMR_NOTIFY, 4, 5, client, 100, 1), (abi.FSMR_NOTIFY, 1, 6, client, 999, 0),
            (abi.FSMR_APPLY, 1, 7, 0, 7, 6), (abi.FSMR_APPLY, 1, 6, 0, 6, 5), (abi.FSMR_APPLY, 1, 8, 0, 8, 7),
            (abi.FSMR_APPLY, 1, 5, 0, 5, 4), (abi.FSMR_APPLY, 1, 0, 0, 0, 0),
            (abi.FSMR_PATTERN, 10, 0, 0, 0b101111, 0)]    # positions 0-3 and 5 are the Notifies
    for k, (kind, cnt, id0, addr, tok0, stride) in enumerate(recs):
        struct.pack_into("<4I", blob, fs_at + (2 * k) * plane * 16, 0, kind | (cnt << 8), id0, addr)
        struct.pack_into("<2Q", blob, fs_at + (2 * k + 1) * plane * 16, tok0, stride)
    struct.pack_into("<2I", blob, fc_at, len(recs), 10)
    eng.restore(bytes(blob))
    ins = eng.drain_fsm()
    runs, batch = eng.fsm_responses()
    records = []
    for kind, cnt, id0, addr, tok0, stride in recs:
        rc = abi.FsmRecord()
        rc.group, rc.hdr, rc.id0, rc.addr, rc.tok0, rc.stride = 0, kind | (cnt << 8), id0, addr, tok0, stride
        records.append(rc)
    want = DriverRef().feed(expand_records(eng._lib, records, 1, 1))
    assert [(f.kind, f.block.id) for f in ins] == [(1, 5), (1, 6), (1, 7), (1, 8), (0, 7), (1, 6), (0, 6), (0, 8), (0, 5), (0, 0)]
    assert expand_responses(runs) == want == [(0, 1, Address.client(), t, i) for i, t in ((7, 102), (6, 999), (8, 103), (5, 100))]
    assert batch.n_dropped == 0


# ---- 6. every drain path ------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("make,fold", ALL)
def test_every_drain_path(make, fold):
    G, R = 12, 5
    p = Pair(make, G, R, fold=fold, seed=6, chain_capacity=512, fsm_units=128)
    p.bootstrap()
    now = 1100
    for how in ("drain", "discard", "records"):
        p.both("run_tokens", now, 100, strided_tokens(9, G, now // 100))
        now += 900
        p.drain(how=how)
    # three batches outstanding on the asynchronous path: each batch's responses are its own
    lib, h = p.eng._lib, p.eng._h
    wants = []
    for k in range(3):
        p.both("run_tokens", now, 100, strided_tokens(7, G, now // 100))
        now += 700
        assert lib.jr_fsm_records_async(h) == 0
        wants.append(p._expect(p.ora.drain_fsm(cap=p.fsm_cap)))
    for k in range(3):
        ptr, batch = C.POINTER(abi.FsmRecord)(), abi.FsmBatch()
        assert lib.jr_fsm_records_wait(h, C.byref(ptr), C.byref(batch)) == 0
        got, _, _ = p.responses()
        assert got == wants[k] and got
    # a capturing step drains too (and discards nothing the oracle hands out)
    p.both("run_tokens", now, 100, strided_tokens(5, G, now // 100))
    p.step(now + 500)


# ---- 7. limits ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("make,fold", ALL)
def test_pending_runs_overflow_drops_never_lies(make, fold):
    G, R = 4, 3
    rng = random.Random(3)
    p = Pair(make, G, R, fold=fold, seed=8, chain_capacity=512, fsm_units=256)
    p.bootstrap()
    for api in (p.eng, p.ora):
        for g in range(G):
            for n in range(2, R + 1):
                api.set_alive(g, n, False)
    p.both("run_tokens", 1100, 100, [[rng.getrandbits(60) | 1 for _ in range(G)] for _ in range(40)])
    got, want, runs, batch = p.drain(strict=False)
    assert batch.n_dropped > 0 and got == want == []
    ptr, b2 = C.POINTER(abi.FsmRecord)(), abi.FsmBatch()
    assert p.eng._fn("fsm_responses")(p.eng._h, C.byref(ptr), C.byref(b2)) == abi.E_CAPACITY
    dropped = batch.n_dropped
    for api in (p.eng, p.ora):
        for g in range(G):
            for n in range(2, R + 1):
                api.set_alive(g, n, True)
    seen_e, seen_o = [], []
    for k in range(4):
        p.both("run", 5100 + 2000 * k, 100, 20, 0)
        got, want, _, batch = p.drain(strict=False)
        dropped += batch.n_dropped
        seen_e += got
        seen_o += want
    assert set(seen_e) <= set(seen_o) and len(seen_e) == len(set(seen_e))
    assert len(seen_o) - len(seen_e) <= dropped and len(seen_o) >= G * 40


@pytest.mark.parametrize("make,fold", ALL)
def test_full_record_fifo_clears_the_map(make, fold):
    G, R = 4, 3
    rng = random.Random(4)
    p = Pair(make, G, R, fold=fold, seed=8, chain_capacity=512, fsm_units=8)
    p.bootstrap()
    p.both("run_tokens", 1100, 100, [[rng.getrandbits(60) | 1 for _ in range(G)] for _ in range(30)])
    ins = p.ora.drain_fsm(cap=p.fsm_cap)
    p.eng.discard_fsm(strict=False)
    runs, batch = p.eng.fsm_responses()
    assert p.ref.feed(ins) and runs == []                   # the reference answers; the engine lost records: nothing
    p.ref.clear()                                           # what the engine's maps now hold
    p.both("run_tokens", 4100, 100, strided_tokens(2, G, 50))
    p.both("run", 4300, 100, 6, 0)
    p.drain()


# ---- 8. random scripts --------------------------------------------------------------------------------------------------

def _random_script(make, fold, seed, rounds=8):
    rng = random.Random(seed)
    G, R = rng.choice([(40, 3), (33, 5), (24, 7)])
    p = Pair(make, G, R, fold=fold, check_batched_driver=False, seed=seed, chain_capacity=512, fsm_units=512,
             fsm_host_records=G * R * 1024, heartbeat_ms=rng.choice([100, 99, 250]))
    p.bootstrap(node=rng.choice([1, 2]))
    now, tick = 1100, 11
    for rnd in range(rounds):
        kind = rng.choice(["run", "tokens", "token_runs", "proposals"])
        ticks = rng.choice([2, 3, 7, 16, 21, 33])
        if kind == "run":
            p.both("run", now, 100, ticks, rng.choice([0, 1, 2]))
        elif kind == "tokens":
            toks = strided_tokens(ticks, G, tick)
            toks = [[t if rng.random() < 0.8 else 0 for t in row] for row in toks]
            p.both("run_tokens", now, 100, toks)
        elif kind == "token_runs":
            p.both("run_token_runs", now, 100, ticks, [(((rnd + 1) << 44) + g + 1, rng.choice([1, 1 << 32])) for g in range(G)])
        else:
            props = [[(rng.choice([1, 1, 2, 0, R]), 9000 + 1000 * rnd + 37 * k + g) for g in range(G)] for k in range(ticks)]
            p.both("run_proposals", now, 100, props)
        now += 100 * ticks
        tick += ticks
        p.drain(how=rng.choice(["drain", "discard", "records"]))
        r = rng.random()
        if r < 0.2:
            assert len(set(p.both("kill_leaders", seed * 31 + rnd, 300))) == 1
        elif r < 0.4:
            g, node, alive = rng.randrange(G), rng.randrange(1, R + 1), rng.random() < 0.4
            p.both("set_alive", g, node, alive)
        elif r < 0.5:
            p.both("truncate", 4)
        if rng.random() < 0.5:
            p.both("leader_table")


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("fold", FOLDS)
def test_random_scripts_on_device_code(seed, fold):
    _random_script(_emu, fold, seed)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [100, 101])
@pytest.mark.parametrize("fold", FOLDS)
def test_random_scripts_on_gpu(seed, fold):
    _random_script(_gpu, fold, seed, rounds=12)


# ---- 9. flag off --------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("make", [pytest.param(_emu, id="emu"), pytest.param(_gpu, id="gpu", marks=pytest.mark.gpu)])
def test_flag_off_and_flag_requirements(make):
    from josefine_b200 import RaftError
    plain = make(8, 3, flags=CAP)
    plain.discard_fsm()
    with pytest.raises(RaftError) as ei:
        plain.fsm_responses()
    assert ei.value.status == abi.E_INVAL
    with pytest.raises(RaftError) as ei:
        make(8, 3, flags=RESP)                                  # requires JR_F_CAPTURE_FSM
    assert ei.value.status == abi.E_INVAL
    # the checkpoint grows by exactly the one segment of maps; without the flag it is what it was
    with_flag = make(8, 3, flags=CAP | RESP)
    plane = 3 * 32                                              # R x groups padded to 32
    seg = (2 * abi.NOTIFY_RUNS * plane + (plane + 3) // 4 + plane) * 16     # runs, run counts, restart marks
    assert len(with_flag.save()) - len(plain.save()) == seg


# ---- 10. full size, GPU -------------------------------------------------------------------------------------------------

_INSTR = np.dtype([("group", "<u4"), ("node", "<u4"), ("kind", "u1"), ("ck", "u1"), ("res", "<u2"), ("cid", "<u4"),
                   ("id", "<u8"), ("next", "<u8"), ("data", "<u8")])
_REC = np.dtype([("group", "<u4"), ("hdr", "<u4"), ("id0", "<u4"), ("addr", "<u4"), ("tok0", "<u8"), ("stride", "<u8")])


def _driver_np(ins, R, pending):
    """DriverRef over one drain's Instructions, vectorised: per (replica, block id), an Apply answers when the event right
    before it is a Notify.  Returns (responses [rep, addr, token, id] in apply order per replica, pending Notifies)."""
    keep = (ins["kind"] == abi.FSM_NOTIFY) | (ins["id"] != 0)
    ins = ins[keep]
    rep = ins["group"].astype(np.int64) * R + ins["node"] - 1
    seq = np.arange(len(ins), dtype=np.int64)
    addr = (ins["ck"].astype(np.uint64) << np.uint64(16)) | ins["cid"].astype(np.uint64)
    ev = dict(rep=np.concatenate([pending["rep"], rep]), id=np.concatenate([pending["id"], ins["id"]]),
              seq=np.concatenate([pending["seq"], seq]), note=np.concatenate([pending["note"], ins["kind"] == abi.FSM_NOTIFY]),
              addr=np.concatenate([pending["addr"], addr]), tok=np.concatenate([pending["tok"], ins["data"]]))
    o = np.lexsort((ev["seq"], ev["id"], ev["rep"]))
    ev = {k: v[o] for k, v in ev.items()}
    same = np.zeros(len(o), bool)
    same[1:] = (ev["rep"][1:] == ev["rep"][:-1]) & (ev["id"][1:] == ev["id"][:-1])
    hit = np.zeros(len(o), bool)
    hit[1:] = same[1:] & ~ev["note"][1:] & ev["note"][:-1]
    j = np.nonzero(hit)[0]
    resp = np.stack([ev["rep"][j].astype(np.uint64), ev["addr"][j - 1], ev["tok"][j - 1], ev["id"][j]])
    resp = resp[:, np.lexsort((ev["seq"][j], ev["rep"][j]))]
    last = np.ones(len(o), bool)
    last[:-1] = ~same[1:]
    k = np.nonzero(last & ev["note"])[0]
    pend = {key: v[k] for key, v in ev.items()}
    pend["seq"] = np.full(len(k), -1, np.int64)
    return resp, pend


def _expand_np(ptr, n, R):
    runs = np.frombuffer(C.string_at(ptr, n * 32), dtype=_REC)
    cnt = (runs["hdr"] >> 8).astype(np.int64)
    rep = runs["group"].astype(np.int64) * R + ((runs["hdr"] >> 2) & 7)
    idx = np.repeat(np.arange(len(runs)), cnt)
    off = np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    e = np.stack([rep[idx].astype(np.uint64), runs["addr"][idx].astype(np.uint64),
                  runs["tok0"][idx] + off.astype(np.uint64) * runs["stride"][idx], runs["id0"][idx].astype(np.uint64) + off.astype(np.uint64)])
    return e[:, np.argsort(e[0], kind="stable")]


@pytest.mark.gpu
@pytest.mark.parametrize("fold", FOLDS)
def test_full_size_responses_equal_the_reference_65536x5(fold):
    """jr_run_tokens at 65,536 x 5, four 64-tick launches, the batched drain: the expanded responses equal the Driver
    restatement over the oracle's Instructions for EVERY group, and every request that committed is answered once."""
    from josefine_b200.raft import load_engine_library
    from oracle.restated import load as load_oracle, RestatedCluster
    import os
    G, R, S = 65536, 5, 64
    eng = _gpu(G, R, seed=1, flags=CAP | RESP | (0 if fold else abi.F_NO_SYMMETRIC_FOLD), fsm_units=16, chain_capacity=512)
    ora = RestatedCluster.create(G, R, n_threads=min(16, os.cpu_count() or 1), seed=1, flags=CAP, chain_capacity=512)
    from tests.stream_cases import _bootstrap
    for api in (eng, ora):
        _bootstrap(api, G, R)
        api.run(100, 100, 16, 0)
        api.leader_table()
        api.discard_fsm(strict=False)
    lib, olib = load_engine_library(), load_oracle()
    cap = G * (R + 1) * S + 4 * G * R
    out_o = (abi.FsmInstr * cap)()
    pending = dict(rep=np.zeros(0, np.int64), id=np.zeros(0, np.uint64), seq=np.zeros(0, np.int64), note=np.zeros(0, bool),
                   addr=np.zeros(0, np.uint64), tok=np.zeros(0, np.uint64))
    now, tick, answered = 1700, 0, []
    for launch in range(4):
        toks = ((np.arange(tick + 1, tick + S + 1, dtype=np.uint64)[:, None] << np.uint64(32)) +
                np.arange(1, G + 1, dtype=np.uint64)[None, :]).copy()
        ptr = toks.ctypes.data_as(C.POINTER(C.c_uint64))
        assert lib.jr_run_tokens(eng._h, C.c_uint64(now), C.c_uint32(100), C.c_uint32(S), ptr) == 0
        assert lib.jr_engine_sync(eng._h) == 0
        assert olib.jro_run_tokens(ora._h, C.c_uint64(now), C.c_uint32(100), C.c_uint32(S), ptr) == 0
        for api in (eng, ora):
            api.truncate(8)
        now += 100 * S
        tick += S
        assert lib.jr_fsm_records_async(eng._h) == 0
        recs, batch = C.POINTER(abi.FsmRecord)(), abi.FsmBatch()
        assert lib.jr_fsm_records_wait(eng._h, C.byref(recs), C.byref(batch)) == 0
        resp, rb = C.POINTER(abi.FsmRecord)(), abi.FsmBatch()
        assert lib.jr_fsm_responses(eng._h, C.byref(resp), C.byref(rb)) == 0 and rb.n_dropped == 0
        got = _expand_np(C.cast(resp, C.c_void_p).value, rb.n_records, R)
        n_o = C.c_size_t(0)
        assert olib.jro_drain_fsm(ora._h, out_o, C.c_size_t(cap), C.byref(n_o)) == 0
        want, pending = _driver_np(np.frombuffer(out_o, dtype=_INSTR, count=n_o.value), R, pending)
        assert got.shape == want.shape and np.array_equal(got, want), f"launch {launch}"
        assert len(np.unique(got[0] // R)) == G and rb.n_records <= 2 * G     # every group answers, compactly
        answered.append(got[2])
    toks = np.concatenate(answered)
    assert len(np.unique(toks)) == len(toks) and len(toks) >= G * (4 * S - 8)
