"""The batched drain run as a pipeline (INTEGRATION.md §2a): up to JR_STAGING_DEPTH quanta in flight, each one
jr_run_token_runs / jr_run_tokens + jr_leader_table_async + jr_fsm_records_async, picked up one or two quanta later by
jr_leader_table_wait + jr_fsm_records_wait (+ jr_fsm_responses), on the submitting thread or on a consumer thread.

Every consumed batch is compared with the C++ oracle making the same calls in the same program order: its synchronous
leader_table where the engine calls jr_leader_table_async (routing is stream-ordered), its drain_fsm where the engine
enqueues the batch.  Runs on the device code built for the host (tests/emu) and on the GPU, over both copy paths of the
drain: the copy engine with its speculative size guess (default) and fsm_copy_kernel (JR_FSM_COPY=sm)."""
import ctypes as C
import os
import threading

import numpy as np
import pytest

from josefine_b200 import abi, expand_responses, fsm_tuple
from tests.stream_cases import _bootstrap
from tests.test_client_responses import DriverRef

CAP, RESP = abi.F_CAPTURE_FSM, abi.F_CLIENT_RESPONSES
DEPTH = 3                      # JR_STAGING_DEPTH
DT = 100
TRUNC = 8                      # jr_set_auto_truncate margin
FOLD_THREADS = 4
REC = C.sizeof(abi.FsmRecord)


def _oracle(g, r, **kw):
    from oracle.restated import RestatedCluster
    return RestatedCluster.create(g, r, n_threads=min(16, os.cpu_count() or 1), **kw)


def _emu(g, r, **kw):
    from tests.emu.emu import EmuEngine
    return EmuEngine.create(g, r, **kw)


def _gpu(g, r, **kw):
    from josefine_b200 import RaftEngine
    return RaftEngine.create(g, r, **kw)


def _declare(lib):
    """argtypes of the asynchronous calls (the emulation build's loader declares only what RaftApi uses)."""
    vp = C.c_void_p
    for name, args in {"jr_leader_table_async": [vp, C.POINTER(abi.LeaderEntry)], "jr_leader_table_wait": [vp],
                       "jr_engine_sync": [vp], "jr_host_alloc": [C.c_size_t, C.POINTER(vp)]}.items():
        fn = getattr(lib, name)
        fn.argtypes, fn.restype = args, C.c_int
    lib.jr_host_free.argtypes, lib.jr_host_free.restype = [vp], None


def _ok(st, what):
    if st != abi.OK:
        raise AssertionError(f"{what} returned {abi.STATUS_NAMES[st] if 0 <= st < len(abi.STATUS_NAMES) else st}")


def _first_difference(got, want):
    """Index and both tuples of the first Instruction where two expanded streams differ (for the failure message)."""
    n = C.sizeof(abi.FsmInstr)
    a, b = got.reshape(-1, n), want.reshape(-1, n)
    i = int(np.argmax((a[:min(len(a), len(b))] != b[:min(len(a), len(b))]).any(axis=1)))
    tup = lambda x: fsm_tuple(abi.FsmInstr.from_buffer_copy(x[i].tobytes())) if i < len(x) else None   # noqa: E731
    return i, tup(a), tup(b)


def steady(k, S, G):
    """Quantum k's tokens, one per group-tick with a constant stride (what a host numbering requests sends):
    tick t of group g proposes ((k*S + t + 1) << 32) + g + 1."""
    return dict(base=(np.uint64(k * S + 1) << np.uint64(32)) + np.arange(1, G + 1, dtype=np.uint64), stride=1 << 32)


class Pipeline:
    """One engine driven as INTEGRATION.md §2a drives it -- pinned buffers from jr_host_alloc, DEPTH token and leader-table
    buffers in rotation, auto-truncate on -- and the oracle making the same calls in the same order.  The oracle is
    synchronous, so its calls are logged at submit time and replayed up to a batch's drain when that batch is checked."""

    def __init__(self, make, G, R, S, api="token_runs", resp=False, seed=1, **cfg):
        self.G, self.R, self.S, self.api, self.resp = G, R, S, api, resp
        self.eng = make(G, R, seed=seed, flags=CAP | (RESP if resp else 0), **cfg)
        self.ora = _oracle(G, R, seed=seed, flags=CAP, **cfg)
        self.fsm_cap = self.eng.cfg.fsm_host_records
        self.lib, self.h, self.olib, self.oh = self.eng._lib, self.eng._h, self.ora._lib, self.ora._h
        _declare(self.lib)
        self._pinned = []
        self.tok = [self._alloc(np.uint64, max(S * G, 2 * G)) for _ in range(DEPTH)]
        self.tab = [self._alloc(np.uint8, G * C.sizeof(abi.LeaderEntry)) for _ in range(DEPTH)]
        self.log = []                      # oracle calls not replayed yet; None marks a drain
        self.want_tab = []                 # the oracle's leader table at each quantum's jr_leader_table_async
        self.n_sub = self.n_con = 0
        self.now = 1700
        self.last_taken = 0                # records of the batch taken last: the next speculative copy's guess grows from it
        self.guess_basis = []              # last_taken when each quantum's batch was enqueued
        self.sizes = []                    # records of each taken batch
        self.ref = DriverRef() if resp else None
        self.applied = {1: np.zeros(G * R, np.uint32), FOLD_THREADS: np.zeros(G * R, np.uint32)}
        self.totals = {1: np.zeros(3, np.uint64), FOLD_THREADS: np.zeros(3, np.uint64)}
        self.ocap = G * (R + 1) * (S + 8) + 4096
        self.obuf = (abi.FsmInstr * self.ocap)()

    def _alloc(self, dtype, n):
        p = C.c_void_p()
        _ok(self.lib.jr_host_alloc(n * np.dtype(dtype).itemsize, C.byref(p)), "jr_host_alloc")
        self._pinned.append(p.value)
        return np.ctypeslib.as_array((C.c_uint8 * (n * np.dtype(dtype).itemsize)).from_address(p.value)).view(dtype)

    def close(self):
        if self.eng._h:
            _ok(self.lib.jr_engine_sync(self.h), "jr_engine_sync")
        for p in self._pinned:
            self.lib.jr_host_free(p)
        self._pinned = []

    # -- both sides, synchronous ---------------------------------------------------------------------------------------
    def warm(self):
        """Leaders elected, auto-truncate on, routes announced, start-up Instructions drained: quanta start at 1700 ms."""
        for api in (self.eng, self.ora):
            _bootstrap(api, self.G, self.R)
            api.set_auto_truncate(TRUNC)
            api.run(100, 100, 16, 0)
            api.leader_table()
            api.discard_fsm(strict=False)

    def both(self, name, *a):
        """A call outside the quantum loop (kill_leaders, set_alive): on the engine now, on the oracle in program order."""
        got = getattr(self.eng, name)(*a)

        def replay():
            assert getattr(self.ora, name)(*a) == got, name
        self.log.append(replay)
        return got

    def _ora_table(self):
        arr = (abi.LeaderEntry * self.G)()
        _ok(self.olib.jro_leader_table(self.oh, arr), "jro_leader_table")
        return C.string_at(arr, C.sizeof(arr))

    def _ora_replay(self):
        """Replay the oracle's log up to the next drain marker and drain: the Instructions of the next batch."""
        while True:
            fn = self.log.pop(0)
            if fn is None:
                break
            fn()
        n = C.c_size_t(0)
        _ok(self.olib.jro_drain_fsm(self.oh, self.obuf, C.c_size_t(self.ocap), C.byref(n)), "jro_drain_fsm")
        return n.value

    # -- the engine's pipeline -----------------------------------------------------------------------------------------
    def submit(self, base=None, stride=None, tokens=None):
        """One quantum: S fused ticks (steady: run-length form base/stride -- through jr_run_token_runs, or expanded to
        jr_run_tokens; tokens: an explicit [S][G] array through jr_run_tokens; nothing: a quantum without proposals),
        then jr_leader_table_async and jr_fsm_records_async."""
        assert self.n_sub - self.n_con < DEPTH
        G, S, b = self.G, self.S, self.n_sub % DEPTH
        now = self.now
        self.now += DT * S
        if tokens is None and base is not None and self.api == "tokens":
            tokens = base[None, :] + np.arange(S, dtype=np.uint64)[:, None] * np.uint64(stride)
        if tokens is None and self.api == "token_runs":
            runs = self.tok[b][:2 * G].reshape(G, 2)
            runs[:, 0] = 0 if base is None else base
            runs[:, 1] = 0 if base is None else stride
            saved = runs.copy()
            _ok(self.lib.jr_run_token_runs(self.h, now, DT, S, C.cast(runs.ctypes.data, C.POINTER(abi.TokenRun))),
                "jr_run_token_runs")
            self.log.append(lambda: _ok(self.olib.jro_run_token_runs(self.oh, now, DT, S, C.cast(
                saved.ctypes.data, C.POINTER(abi.TokenRun))), "jro_run_token_runs"))
        else:
            toks = self.tok[b][:S * G].reshape(S, G)
            toks[:] = 0 if tokens is None else tokens
            saved = toks.copy()
            _ok(self.lib.jr_run_tokens(self.h, now, DT, S, C.cast(toks.ctypes.data, C.POINTER(C.c_uint64))),
                "jr_run_tokens")
            self.log.append(lambda: _ok(self.olib.jro_run_tokens(self.oh, now, DT, S, C.cast(
                saved.ctypes.data, C.POINTER(C.c_uint64))), "jro_run_tokens"))
        _ok(self.lib.jr_leader_table_async(self.h, C.cast(self.tab[b].ctypes.data, C.POINTER(abi.LeaderEntry))),
            "jr_leader_table_async")
        self.log.append(lambda: self.want_tab.append(self._ora_table()))
        _ok(self.lib.jr_fsm_records_async(self.h), "jr_fsm_records_async")
        self.log.append(None)
        self.guess_basis.append(self.last_taken)
        self.n_sub += 1

    def take(self):
        """jr_leader_table_wait + jr_fsm_records_wait (+ jr_fsm_responses): the oldest outstanding quantum."""
        k = self.n_con
        _ok(self.lib.jr_leader_table_wait(self.h), "jr_leader_table_wait")
        table = self.tab[k % DEPTH].tobytes()
        recs, batch = C.POINTER(abi.FsmRecord)(), abi.FsmBatch()
        st = self.lib.jr_fsm_records_wait(self.h, C.byref(recs), C.byref(batch))
        assert st == abi.OK and batch.n_dropped == 0, (k, st, batch.n_dropped)
        t = dict(k=k, table=table, recs=recs, batch=batch)
        if self.resp:
            t["resp"], t["rbatch"] = C.POINTER(abi.FsmRecord)(), abi.FsmBatch()
            _ok(self.lib.jr_fsm_responses(self.h, C.byref(t["resp"]), C.byref(t["rbatch"])), "jr_fsm_responses")
        self.last_taken = batch.n_records
        self.sizes.append(batch.n_records)
        self.n_con += 1
        return t

    def read(self, t):
        """What a host does with a taken batch: expand it, fold it (one thread and FOLD_THREADS), read the responses."""
        recs, n = t["recs"], t["batch"].n_records
        need = C.c_size_t(0)
        st = self.lib.jr_fsm_expand(recs, C.c_size_t(n), self.G, self.R, None, C.c_size_t(0), C.byref(need))
        assert st in (abi.OK, abi.E_CAPACITY), st
        out = (abi.FsmInstr * max(need.value, 1))()
        if need.value:
            _ok(self.lib.jr_fsm_expand(recs, C.c_size_t(n), self.G, self.R, out, need, C.byref(need)), "jr_fsm_expand")
        r = dict(k=t["k"], table=t["table"], n_records=n, n_instructions=t["batch"].n_instructions,
                 ins=np.frombuffer(out, np.uint8, count=need.value * C.sizeof(abi.FsmInstr)))
        _ok(self.lib.jr_fsm_fold(C.cast(recs, C.c_void_p), C.c_size_t(n), self.G, self.R, self.applied[1].ctypes.data,
                                 self.totals[1].ctypes.data), "jr_fsm_fold")
        _ok(self.lib.jr_fsm_fold_mt(C.cast(recs, C.c_void_p), C.c_size_t(n), self.G, self.R,
                                    self.applied[FOLD_THREADS].ctypes.data, self.totals[FOLD_THREADS].ctypes.data,
                                    FOLD_THREADS), "jr_fsm_fold_mt")
        r["fold"] = [(self.applied[t].copy(), self.totals[t].copy()) for t in (1, FOLD_THREADS)]
        if self.resp:
            rb = t["rbatch"]
            assert rb.n_dropped == 0
            runs = [abi.FsmRecord.from_buffer_copy(t["resp"][i]) for i in range(rb.n_records)]
            r["responses"] = expand_responses(runs)
            assert rb.n_instructions == len(r["responses"])
        return r

    def check(self, r):
        """Batch r against the oracle replayed up to that batch's drain."""
        k = r["k"]
        n = self._ora_replay()
        want = np.frombuffer(self.obuf, np.uint8, count=n * C.sizeof(abi.FsmInstr))
        assert r["n_instructions"] == n, (k, r["n_instructions"], n)
        if not np.array_equal(r["ins"], want):
            raise AssertionError(f"quantum {k}: expanded records differ from the oracle's Instructions at "
                                 f"{_first_difference(r['ins'], want)}")
        assert r["table"] == self.want_tab[k], f"quantum {k}: leader table differs from the oracle's"
        (a1, t1), (am, tm) = r["fold"]
        assert np.array_equal(a1, am) and np.array_equal(t1, tm), f"quantum {k}: jr_fsm_fold_mt != jr_fsm_fold"
        if self.resp:
            want_resp = self.ref.feed([self.obuf[i] for i in range(n)])
            assert r["responses"] == want_resp, f"quantum {k}: responses differ from the Driver restatement"

    def finish(self):
        assert self.n_con == self.n_sub and not [f for f in self.log if f is not None]
        for f in self.log:
            f()
        self.log = []
        _ok(self.lib.jr_engine_sync(self.h), "jr_engine_sync")
        assert self.eng.state_digest() == self.ora.state_digest()
        rep, findings = self.eng.verify_groups()
        assert findings == [], [(f.group, f.node) for f in findings[:8]]


def drive(p, plan, before=None):
    """The §2a loop at depth 3: quantum k is consumed after k+1 and k+2 have been submitted, and the submitter enqueues
    k+3 right after k's wait returns, while the host still reads k (the header lets it).  plan[k] is submit()'s keyword
    arguments; before[k] runs just before quantum k is submitted."""
    before = before or {}
    n = len(plan)

    def sub(j):
        if j in before:
            before[j](p)
        p.submit(**plan[j])

    for j in range(min(DEPTH, n)):
        sub(j)
    for k in range(n):
        t = p.take()
        if k + DEPTH < n:
            sub(k + DEPTH)
        p.check(p.read(t))


def _copy_params():
    return [pytest.param("dma", id="dma"), pytest.param("sm", id="sm")]


def _set_copy(monkeypatch, copy):
    if copy == "sm":
        monkeypatch.setenv("JR_FSM_COPY", "sm")
    else:
        monkeypatch.delenv("JR_FSM_COPY", raising=False)


def _where():
    return [pytest.param(_emu, id="emu"), pytest.param(_gpu, id="gpu", marks=pytest.mark.gpu)]


# ---- (a) lifetime of a returned batch ----------------------------------------------------------------------------------

@pytest.mark.parametrize("resp", [False, True], ids=["records", "responses"])
@pytest.mark.parametrize("depth", [1, 2, 3])
@pytest.mark.parametrize("copy", _copy_params())
@pytest.mark.parametrize("make", _where())
def test_returned_batch_survives_the_next_enqueue(make, copy, depth, resp, monkeypatch):
    """The header: the records (and responses) jr_fsm_records_wait returns stay valid until the JR_STAGING_DEPTH-1'th
    jr_fsm_records_async after it.  With `depth` batches outstanding at the wait, one more quantum and its enqueue must
    leave the returned bytes untouched, and they must be the oracle's drain of that quantum."""
    _set_copy(monkeypatch, copy)
    G, R, S = 8, 3, 8
    p = Pipeline(make, G, R, S, api="tokens", resp=resp, chain_capacity=256, fsm_units=64)
    try:
        p.warm()
        for k in range(depth):
            p.submit(**steady(k, S, G))
        t = p.take()
        n = t["batch"].n_records
        snap = C.string_at(t["recs"], n * REC)
        if resp:
            n_resp = t["rbatch"].n_records
            snap_resp = C.string_at(t["resp"], n_resp * REC)
            assert n_resp > 0
        p.submit(**steady(depth, S, G))
        _ok(p.lib.jr_engine_sync(p.h), "jr_engine_sync")
        assert n > 0 and C.string_at(t["recs"], n * REC) == snap, f"depth {depth}: the returned records were overwritten"
        if resp:
            assert C.string_at(t["resp"], n_resp * REC) == snap_resp, f"depth {depth}: the returned responses were overwritten"
        p.check(p.read(t))
        while p.n_con < p.n_sub:
            p.check(p.read(p.take()))
        p.finish()
    finally:
        p.close()


# ---- (b) the §2a loop at depth 3 ---------------------------------------------------------------------------------------

def _loop_plan(G, S, n=8):
    """Steady quanta; leaders of ~30% of the groups silenced before quantum 2 (its tokens still go to the old routes: to
    a dead node, then to followers once the silenced leaders are revived before quantum 4); quantum 3 proposes nothing."""
    plan = [steady(k, S, G) for k in range(n)]
    plan[3] = {}
    revive = range(0, G, max(1, G // 64))

    def kill(p):
        assert p.both("kill_leaders", 17, 300) > 0

    def wake(p):
        for g in revive:
            for node in range(1, p.R + 1):
                p.both("set_alive", g, node, True)
    return plan, {2: kill, 4: wake}


@pytest.mark.parametrize("api,resp", [("token_runs", True), ("tokens", False)])
@pytest.mark.parametrize("R", [3, 5])
@pytest.mark.parametrize("G", [33, 96])
@pytest.mark.parametrize("copy", _copy_params())
def test_pipelined_loop_on_device_code(copy, G, R, api, resp, monkeypatch):
    _set_copy(monkeypatch, copy)
    S = 16
    p = Pipeline(_emu, G, R, S, api=api, resp=resp, seed=G + R, chain_capacity=256, fsm_units=4 * S + 64)
    try:
        p.warm()
        plan, before = _loop_plan(G, S)
        drive(p, plan, before)
        p.finish()
    finally:
        p.close()


@pytest.mark.gpu
@pytest.mark.parametrize("G,api,copy", [(4096, "token_runs", "dma"), (4096, "token_runs", "sm"), (4096, "tokens", "dma"),
                                        (4096, "tokens", "sm"), (65536, "token_runs", "dma"), (65536, "tokens", "sm")])
def test_pipelined_loop_on_gpu(G, api, copy, monkeypatch):
    """4,096 x 5 and 65,536 x 5, 64-tick quanta: batches of 4,096 records and more, so jr_fsm_fold_mt folds on threads."""
    _set_copy(monkeypatch, copy)
    R, S = 5, 64
    p = Pipeline(_gpu, G, R, S, api=api, seed=3, chain_capacity=512, fsm_units=2 * S + 32, fsm_host_records=4 * G * R)
    try:
        p.warm()
        plan, before = _loop_plan(G, S, n=6)
        drive(p, plan, before)
        assert max(p.sizes) >= 4096
        p.finish()
    finally:
        p.close()


# ---- (c) the speculative copy's tail under the pipeline ----------------------------------------------------------------

def _guess(p, k):
    """fsm_records_enqueue's speculative copy size for quantum k's batch."""
    prev = p.guess_basis[k]
    return min(p.fsm_cap, max(prev + prev // 8 + 1024, 16384))


def _tail_plan(G, S, n, at, seed):
    rng = np.random.default_rng(seed)
    plan = [steady(k, S, G) for k in range(n)]
    plan[at] = dict(tokens=rng.integers(1, 1 << 63, size=(S, G), dtype=np.uint64))    # arbitrary: no runs to speak of
    return plan


@pytest.mark.parametrize("copy", _copy_params())
@pytest.mark.parametrize("make", _where())
def test_batch_larger_than_the_copy_guess(make, copy, monkeypatch):
    """After constant-stride quanta (a few records per replica), a quantum of arbitrary tokens (no constant stride to
    run-length encode) with two other batches outstanding: its batch outgrows the speculative copy, whose tail
    fsm_records_take fetches -- the batch must still be the oracle's."""
    _set_copy(monkeypatch, copy)
    G, R, S, AT = 384, 5, 48, 4          # ~1.5 records per group-tick of arbitrary tokens: ~27,000 records > 16,384
    p = Pipeline(make, G, R, S, api="token_runs", resp=True, seed=9, chain_capacity=256, fsm_units=4 * S + 64,
                 fsm_host_records=G * (R + 1) * S + 4096)
    try:
        p.warm()
        drive(p, _tail_plan(G, S, AT + 3, AT, seed=9))
        assert p.sizes[AT] > _guess(p, AT), (p.sizes, _guess(p, AT))
        p.finish()
    finally:
        p.close()


# ---- (d) two host threads ----------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("copy", _copy_params())
def test_consumer_thread_on_gpu(copy, monkeypatch):
    """A consumer thread waits for, expands, folds and reads the responses of quantum k while the submitting thread
    enqueues quantum k+3: the header lets the submitter go on as soon as k's wait has returned, and asks only that the
    consumer be done with k before the submitter's second enqueue after that wait (k+4).  Includes a quantum that
    outgrows the speculative copy.  Every batch is checked against the oracle afterwards, over the same call log."""
    _set_copy(monkeypatch, copy)
    G, R, S, N, AT = 4096, 5, 32, 10, 5
    p = Pipeline(_gpu, G, R, S, api="token_runs", resp=True, seed=5, chain_capacity=512, fsm_units=4 * S + 64,
                 fsm_host_records=G * (R + 1) * S + 4096)
    try:
        p.warm()
        plan = _tail_plan(G, S, N, AT, seed=5)
        ready, taken, done = threading.Semaphore(0), threading.Semaphore(0), threading.Semaphore(0)
        failed, results = [], [None] * N

        def consumer():
            try:
                for k in range(N):
                    ready.acquire()                  # (a wait with nothing outstanding is JR_E_INVAL, not a block)
                    t = p.take()
                    taken.release()
                    results[k] = p.read(t)
                    done.release()
            except BaseException as ex:      # noqa: BLE001 -- handed to the submitting thread
                failed.append(ex)
                for _ in range(2 * N):
                    taken.release()
                    done.release()

        th = threading.Thread(target=consumer, name="fsm-driver")
        th.start()
        try:
            for j in range(N):
                if j >= DEPTH:
                    taken.acquire()          # batch j-3 has been returned: at most two outstanding
                if j >= DEPTH + 1:
                    done.acquire()           # batch j-4 has been read: its buffer may be reused from this enqueue on
                if failed:
                    break
                p.submit(**plan[j])
                ready.release()
        finally:
            for _ in range(N):               # (only a consumer still waiting after a failure takes these)
                ready.release()
            th.join()
        if failed:
            raise failed[0]
        for r in results:
            p.check(r)
        basis = max(p.sizes[:AT])
        assert p.sizes[AT] > min(p.fsm_cap, max(basis + basis // 8 + 1024, 16384)), p.sizes
        p.finish()
    finally:
        p.close()


# ---- (e) a caller's stream ---------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_pipelined_loop_on_a_caller_stream():
    """jr_engine_set_stream: the loop on a torch stream, back to the engine's own stream (NULL) while batches are
    outstanding; jr_leader_table_device into a torch tensor equals jr_leader_table and the oracle's table."""
    import torch
    G, R, S = 4096, 5, 32
    p = Pipeline(_gpu, G, R, S, api="token_runs", seed=7, chain_capacity=512, fsm_units=2 * S + 32,
                 fsm_host_records=4 * G * R)
    try:
        p.warm()
        stream = torch.cuda.Stream()
        p.eng.set_stream(stream.cuda_stream)
        plan, before = _loop_plan(G, S, n=6)
        before[3] = lambda p: p.eng.set_stream(0)
        drive(p, plan, before)
        dev = torch.zeros(G * C.sizeof(abi.LeaderEntry), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()                                   # (the engine's own stream does not wait for torch's)
        p.eng.leader_table_device(dev.data_ptr())
        host = (abi.LeaderEntry * G)()
        _ok(p.lib.jr_leader_table(p.h, host), "jr_leader_table")
        p.eng.sync()
        torch.cuda.synchronize()
        assert bytes(dev.cpu().numpy()) == C.string_at(host, C.sizeof(host))
        p.finish()
        assert C.string_at(host, C.sizeof(host)) == p._ora_table()    # (also the oracle's announce matching the two above)
        p.eng.set_stream(stream.cuda_stream)
        drive(p, [steady(k, S, G) for k in range(6, 10)])
        p.finish()
    finally:
        p.close()


# ---- (f) bookkeeping -----------------------------------------------------------------------------------------------------

def test_staging_bookkeeping_on_device_code():
    """The FIFO's limits: a fourth outstanding batch, a wait with nothing outstanding, the synchronous drains while
    batches are outstanding (a capturing jr_step still steps); a leader-table wait with nothing pending; FIFO order."""
    from josefine_b200 import RaftError
    from tests import parity
    G, R, S = 8, 3, 8
    p = Pipeline(_emu, G, R, S, api="tokens", chain_capacity=256, fsm_units=64)
    try:
        p.warm()
        lib, h = p.lib, p.h
        recs, batch = C.POINTER(abi.FsmRecord)(), abi.FsmBatch()
        assert lib.jr_fsm_records_wait(h, C.byref(recs), C.byref(batch)) == abi.E_INVAL
        assert lib.jr_leader_table_wait(h) == abi.OK
        for k in range(DEPTH):
            p.submit(**steady(k, S, G))
        assert lib.jr_fsm_records_async(h) == abi.E_INVAL
        n = C.c_size_t(0)
        assert lib.jr_drain_fsm(h, None, C.c_size_t(0), C.byref(n)) == abi.E_INVAL
        with pytest.raises(RaftError) as ei:
            p.eng.step(p.now)
        assert ei.value.status == abi.E_INVAL
        for k in range(DEPTH):                                     # FIFO: quantum k's batch comes back k-th
            p.check(p.read(p.take()))
        assert lib.jr_fsm_records_wait(h, C.byref(recs), C.byref(batch)) == abi.E_INVAL
        assert lib.jr_leader_table_wait(h) == abi.OK             # (each take waited for its quantum's table)
        p.ora.step(p.now)                                          # the engine's step ran although its capture failed
        parity.compare_states(p.eng, p.ora, chain_ids=16)
        p.eng.discard_fsm()                                        # (the failed capture left the step's Instructions)
        p.finish()
    finally:
        p.close()
