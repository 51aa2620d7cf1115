"""Host-side mirror of josefine's Raft step interface over the C ABI.

Names follow the reference (tychedelia/josefine, src/raft):

  Command.*            -> enum Command                      src/raft/mod.rs:160-227
  Address              -> enum Address                      src/raft/rpc.rs:5-14
  RaftEngine           -> G x R batched RaftHandle          src/raft/mod.rs:417-435
  RaftEngine.step      -> Apply::apply per replica          src/raft/mod.rs:483-489
  ReplicaHandle        -> RaftHandle accessors              src/raft/mod.rs:437-468

`RaftApi` is written against a (library, prefix) pair so the test oracle
(oracle/restated.py, prefix "jro_") can be driven by exactly the same calls;
this module itself never imports or loads anything under oracle/.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass
from typing import Iterable, List, Optional, Sequence, Tuple

from . import abi


class RaftError(RuntimeError):
    def __init__(self, status: int, where: str, detail: str = ""):
        name = abi.STATUS_NAMES[status] if 0 <= status < len(abi.STATUS_NAMES) else str(status)
        super().__init__(f"{where}: {name}{(' - ' + detail) if detail else ''}")
        self.status = status


@dataclass(frozen=True)
class Address:
    """src/raft/rpc.rs:5-14"""
    kind: int
    id: int = 0

    @staticmethod
    def peers() -> "Address":
        return Address(abi.ADDR_PEERS)

    @staticmethod
    def peer(node: int) -> "Address":
        return Address(abi.ADDR_PEER, node)

    @staticmethod
    def local() -> "Address":
        return Address(abi.ADDR_LOCAL)

    @staticmethod
    def client() -> "Address":
        return Address(abi.ADDR_CLIENT)


class Command:
    """Constructors for the reference's Command variants as jr_msg (mod.rs:160-227).

    `group` and `to` say which replica applies it (`raft.apply(cmd)` in the
    reference); `from_` is informational, as in rpc.rs:17-21.
    """

    @staticmethod
    def _base(group: int, to: int, kind: int, from_: int = 0) -> abi.Msg:
        m = abi.Msg()
        m.group = group
        m.to_kind = abi.ADDR_PEER
        m.to_id = to
        m.from_kind = abi.ADDR_PEER if from_ else abi.ADDR_LOCAL
        m.from_id = from_
        m.kind = kind
        return m

    @staticmethod
    def tick(group: int, to: int) -> abi.Msg:
        return Command._base(group, to, abi.CMD_TICK)

    @staticmethod
    def timeout(group: int, to: int) -> abi.Msg:
        return Command._base(group, to, abi.CMD_TIMEOUT)

    @staticmethod
    def noop(group: int, to: int) -> abi.Msg:
        return Command._base(group, to, abi.CMD_NOOP)

    @staticmethod
    def vote_request(group: int, to: int, term: int, candidate_id: int, last_term: int, head: int) -> abi.Msg:
        m = Command._base(group, to, abi.CMD_VOTE_REQUEST, candidate_id)
        m.term, m.node_id, m.last_term, m.block = term, candidate_id, last_term, head
        return m

    @staticmethod
    def vote_response(group: int, to: int, term: int, from_: int, granted: bool) -> abi.Msg:
        m = Command._base(group, to, abi.CMD_VOTE_RESPONSE, from_)
        m.term, m.node_id, m.flag = term, from_, int(granted)
        return m

    @staticmethod
    def append_entries(group: int, to: int, term: int, leader_id: int,
                       blocks: Sequence[Tuple[int, int, int]] = ()) -> abi.Msg:
        if len(blocks) > abi.MAX_AE_BLOCKS:
            raise ValueError("at most MAX_INFLIGHT=5 blocks per AppendEntries (progress.rs:117)")
        m = Command._base(group, to, abi.CMD_APPEND_ENTRIES, leader_id)
        m.term, m.node_id, m.n_blocks = term, leader_id, len(blocks)
        for i, b in enumerate(blocks):
            bid, nxt = b[0], b[1]
            data = b[2] if len(b) > 2 else 0
            m.blocks[i].id, m.blocks[i].next, m.blocks[i].data = bid, nxt, data
        return m

    @staticmethod
    def append_response(group: int, to: int, node_id: int, term: int, head: int, success: bool = True) -> abi.Msg:
        m = Command._base(group, to, abi.CMD_APPEND_RESPONSE, node_id)
        m.node_id, m.term, m.block, m.flag = node_id, term, head, int(success)
        return m

    @staticmethod
    def heartbeat(group: int, to: int, term: int, commit: int, leader_id: int) -> abi.Msg:
        m = Command._base(group, to, abi.CMD_HEARTBEAT, leader_id)
        m.term, m.block, m.node_id = term, commit, leader_id
        return m

    @staticmethod
    def heartbeat_response(group: int, to: int, commit: int, has_committed: bool, from_: int = 0) -> abi.Msg:
        m = Command._base(group, to, abi.CMD_HEARTBEAT_RESPONSE, from_)
        m.block, m.flag = commit, int(has_committed)
        return m

    @staticmethod
    def client_request(group: int, to: int, token: int, address: Address = Address.client()) -> abi.Msg:
        m = Command._base(group, to, abi.CMD_CLIENT_REQUEST)
        m.token, m.client_kind, m.client_id = token, address.kind, address.id
        return m

    @staticmethod
    def client_response(group: int, to: int, token: int) -> abi.Msg:
        m = Command._base(group, to, abi.CMD_CLIENT_RESPONSE)
        m.token = token
        return m


def msg_tuple(m: abi.Msg) -> tuple:
    """Canonical comparable form of a Message (all ABI fields)."""
    return (m.group, m.from_kind, m.from_id, m.to_kind, m.to_id, m.kind, m.flag, m.node_id, m.term,
            m.last_term, m.block, m.token, m.client_kind, m.client_id, m.n_blocks,
            tuple((m.blocks[i].id, m.blocks[i].next, m.blocks[i].data) for i in range(m.n_blocks)))


def fsm_tuple(f: abi.FsmInstr) -> tuple:
    return (f.group, f.node, f.kind, f.client_kind, f.client_id, f.block.id, f.block.next, f.block.data)


DEFAULT_CAPTURE_CAP = 1 << 18


@dataclass
class StepResult:
    messages: List[abi.Msg]
    fsm: List[abi.FsmInstr]
    n_faulted: Optional[int] = None      # with report_faults: replicas holding a sticky fault after the step


class RaftApi:
    """Thin object wrapper over one (library, prefix) implementation of the C ABI."""

    def __init__(self, lib: C.CDLL, prefix: str, handle: C.c_void_p, cfg: abi.Config):
        self._lib, self._p, self._h, self.cfg = lib, prefix, handle, cfg
        self.n_groups, self.n_replicas = cfg.n_groups, cfg.n_replicas

    # -- plumbing ---------------------------------------------------------------
    def _fn(self, name: str):
        return getattr(self._lib, self._p + name)

    def _check(self, status: int, where: str):
        if status != abi.OK:
            detail = ""
            if self._p == "jr_":
                self._lib.jr_last_error.restype = C.c_char_p
                detail = (self._lib.jr_last_error() or b"").decode()
            raise RaftError(status, self._p + where, detail)

    def close(self):
        if self._h:
            self._fn("destroy" if self._p == "jro_" else "engine_destroy")(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- stepping ---------------------------------------------------------------
    def step(self, now_ms: int, flags: int = abi.STEP_DELIVER | abi.STEP_TICK,
             inject: Iterable[abi.Msg] = (), proposals: Optional[Sequence[Tuple[int, int]]] = None,
             n_synth: int = 0, cap_msgs: Optional[int] = None, cap_fsm: Optional[int] = None,
             report_faults: bool = False) -> StepResult:
        """One jr_step.  `proposals` is a per-group list of (node, token); node 0 = none."""
        a = abi.StepArgs()
        a.now_ms, a.flags, a.n_synth = now_ms, flags, n_synth
        if n_synth:
            a.flags |= abi.STEP_SYNTH_PROPOSALS
        if report_faults:
            a.flags |= abi.STEP_REPORT_FAULTS
        inj = list(inject)
        if inj:
            arr = (abi.Msg * len(inj))(*inj)
            a.inject, a.n_inject = arr, len(inj)
        if proposals is not None:
            if len(proposals) != self.n_groups:
                raise ValueError("proposals must have one entry per group")
            parr = (abi.Proposal * self.n_groups)()
            for g, (node, token) in enumerate(proposals):
                parr[g].node, parr[g].token = node, token
            a.proposals = parr
        cap_m = cap_f = 0
        # default capture buffers: the worst case, but never more than DEFAULT_CAPTURE_CAP entries
        # (capture is a debugging / small-deployment feature; pass cap_msgs / cap_fsm to go beyond)
        if self.cfg.flags & abi.F_CAPTURE_MESSAGES:
            cap_m = cap_msgs if cap_msgs is not None else min(
                self.n_groups * self.n_replicas * self.cfg.mailbox_units, DEFAULT_CAPTURE_CAP)
            mbuf = (abi.Msg * max(cap_m, 1))()
            a.out_msgs, a.cap_msgs = mbuf, cap_m
        if self.cfg.flags & abi.F_CAPTURE_FSM:
            cap_f = cap_fsm if cap_fsm is not None else min(
                self.n_groups * self.n_replicas * self.cfg.fsm_units, DEFAULT_CAPTURE_CAP)
            fbuf = (abi.FsmInstr * max(cap_f, 1))()
            a.out_fsm, a.cap_fsm = fbuf, cap_f
        st = self._fn("step")(self._h, C.byref(a))
        if st == abi.E_CAPACITY:
            raise RaftError(st, self._p + "step", f"the step emitted {a.n_msgs} messages / {a.n_fsm} instructions but the "
                            f"capture buffers hold {cap_m} / {cap_f}; the step HAS been applied -- pass cap_msgs / cap_fsm")
        self._check(st, "step")
        msgs = [mbuf[i] for i in range(a.n_msgs)] if cap_m else []
        fsm = [fbuf[i] for i in range(a.n_fsm)] if cap_f else []
        return StepResult(msgs, fsm, a.n_faulted if report_faults else None)

    def apply(self, cmd: abi.Msg, now_ms: int = 0) -> StepResult:
        """`raft.apply(cmd)` on one replica: no mail delivery, no implicit Tick."""
        return self.step(now_ms, flags=0, inject=[cmd])

    def run(self, now0_ms: int, dt_ms: int, n_steps: int, n_synth: int = 0):
        self._check(self._fn("run")(self._h, C.c_uint64(now0_ms), C.c_uint32(dt_ms), C.c_uint32(n_steps),
                                    C.c_uint32(n_synth)), "run")

    def run_proposals(self, now0_ms: int, dt_ms: int, proposals: Sequence[Sequence[Tuple[int, int]]], flags: int = 0):
        """Fused ticks with client input: proposals[k][g] = (node, token) for tick k (node 0 = none)."""
        n = len(proposals)
        arr = (abi.Proposal * (n * self.n_groups))()
        for k, tick in enumerate(proposals):
            if len(tick) != self.n_groups:
                raise ValueError("every tick needs one proposal entry per group")
            for g, (node, token) in enumerate(tick):
                arr[k * self.n_groups + g].node, arr[k * self.n_groups + g].token = node, token
        self._check(self._fn("run_proposals")(self._h, C.c_uint64(now0_ms), C.c_uint32(dt_ms), C.c_uint32(n), arr,
                                              C.c_uint32(flags)), "run_proposals")
        if self._p == "jr_":
            self._check(self._lib.jr_engine_sync(self._h), "engine_sync")   # `arr` is pageable and about to be freed

    def run_tokens(self, now0_ms: int, dt_ms: int, tokens: Sequence[Sequence[int]]):
        """Fused ticks with leader-routed client input: tokens[k][g] (0 = none) is proposed at the node the last
        leader_table() call announced as group g's leader."""
        n = len(tokens)
        arr = (C.c_uint64 * max(n * self.n_groups, 1))()
        for k, tick in enumerate(tokens):
            if len(tick) != self.n_groups:
                raise ValueError("every tick needs one token per group")
            arr[k * self.n_groups:(k + 1) * self.n_groups] = list(tick)
        self._check(self._fn("run_tokens")(self._h, C.c_uint64(now0_ms), C.c_uint32(dt_ms), C.c_uint32(n), arr), "run_tokens")
        if self._p == "jr_":
            self._check(self._lib.jr_engine_sync(self._h), "engine_sync")   # `arr` is pageable and about to be freed

    def drain_fsm(self, cap: Optional[int] = None) -> List[abi.FsmInstr]:
        n = C.c_size_t(0)
        if cap is None:
            cap = min(self.n_groups * self.n_replicas * self.cfg.fsm_units, 4 * DEFAULT_CAPTURE_CAP)
        buf = (abi.FsmInstr * max(cap, 1))()
        self._check(self._fn("drain_fsm")(self._h, buf, C.c_size_t(cap), C.byref(n)), "drain_fsm")
        return [buf[i] for i in range(n.value)]

    def run_token_runs(self, now0_ms: int, dt_ms: int, n_steps: int, runs: Sequence[Tuple[int, int]]):
        """jr_run_token_runs: group g proposes base + k * stride at tick k (base 0 = nothing), routed like run_tokens."""
        if len(runs) != self.n_groups:
            raise ValueError("one (base, stride) run per group")
        arr = (abi.TokenRun * self.n_groups)()
        for g, (base, stride) in enumerate(runs):
            arr[g].base, arr[g].stride = base, stride
        self._check(self._fn("run_token_runs")(self._h, C.c_uint64(now0_ms), C.c_uint32(dt_ms), C.c_uint32(n_steps), arr), "run_token_runs")
        if self._p == "jr_":
            self._check(self._lib.jr_engine_sync(self._h), "engine_sync")   # `arr` is pageable and about to be freed

    def discard_fsm(self, strict: bool = True) -> int:
        """Drain without returning the Instructions; their number.  strict=False: records lost to a full FIFO are not an
        error (start-up phases a caller does not care about)."""
        n = C.c_size_t(0)
        st = self._fn("drain_fsm")(self._h, None, C.c_size_t(0), C.byref(n))
        if not (st == abi.E_CAPACITY and not strict):
            self._check(st, "drain_fsm")
        return n.value

    def fsm_records(self) -> Tuple[List[abi.FsmRecord], abi.FsmBatch]:
        """jr_fsm_records_async + jr_fsm_records_wait: everything accumulated since the last drain, compact form
        (copied out of the engine's pinned buffer)."""
        self._check(self._fn("fsm_records_async")(self._h), "fsm_records_async")
        ptr, batch = C.POINTER(abi.FsmRecord)(), abi.FsmBatch()
        st = self._fn("fsm_records_wait")(self._h, C.byref(ptr), C.byref(batch))
        if st not in (abi.OK, abi.E_CAPACITY):
            self._check(st, "fsm_records_wait")
        recs = [abi.FsmRecord.from_buffer_copy(ptr[i]) for i in range(batch.n_records)]
        if st == abi.E_CAPACITY:
            raise RaftError(st, self._p + "fsm_records_wait", f"{batch.n_dropped} records dropped")
        return recs, batch

    def fsm_responses(self) -> Tuple[List[abi.FsmRecord], abi.FsmBatch]:
        """jr_fsm_responses (F_CLIENT_RESPONSES): the ClientResponse runs of the batch most recently taken (by
        fsm_records, drain_fsm, discard_fsm or a capturing step), copied out of the engine's pinned buffer.  Runs the
        engine could not produce are counted in batch.n_dropped (the call's JR_E_CAPACITY) and are not an error here."""
        ptr, batch = C.POINTER(abi.FsmRecord)(), abi.FsmBatch()
        st = self._fn("fsm_responses")(self._h, C.byref(ptr), C.byref(batch))
        if st != abi.E_CAPACITY:
            self._check(st, "fsm_responses")
        return [abi.FsmRecord.from_buffer_copy(ptr[i]) for i in range(batch.n_records)], batch

    def fsm_expand(self, records: Sequence[abi.FsmRecord]) -> List[abi.FsmInstr]:
        """jr_fsm_expand (pure host code of the engine library): records -> Instructions in jr_step order."""
        return expand_records(self._lib, records, self.n_groups, self.n_replicas)

    # -- introspection ------------------------------------------------------------
    def query_many(self, targets: Sequence[Tuple[int, int]]) -> List[abi.ReplicaState]:
        """jr_query_many: one kernel + one copy for all (group, node) targets."""
        n = len(targets)
        if not hasattr(self._lib, self._p + "query_many"):
            return [self.query(g, nd) for g, nd in targets]
        gs = (C.c_uint32 * max(n, 1))(*[t[0] for t in targets])
        ns = (C.c_uint32 * max(n, 1))(*[t[1] for t in targets])
        out = (abi.ReplicaState * max(n, 1))()
        self._check(self._fn("query_many")(self._h, gs, ns, C.c_size_t(n), out), "query_many")
        return [out[i] for i in range(n)]

    def chain_read_many(self, reqs: Sequence[Tuple[int, int, int, int]]) -> List[List[Optional[Tuple[int, int, int]]]]:
        """jr_chain_read_many: reqs = (group, node, first_id, count); one kernel + one copy."""
        if not hasattr(self._lib, self._p + "chain_read_many"):
            return [self.chain_read(*r) for r in reqs]
        n = len(reqs)
        total = sum(r[3] for r in reqs)
        gs = (C.c_uint32 * max(n, 1))(*[r[0] for r in reqs])
        ns = (C.c_uint32 * max(n, 1))(*[r[1] for r in reqs])
        fs = (C.c_uint64 * max(n, 1))(*[r[2] for r in reqs])
        cs = (C.c_uint32 * max(n, 1))(*[r[3] for r in reqs])
        out = (abi.Block * max(total, 1))()
        present = (C.c_uint8 * max(total, 1))()
        self._check(self._fn("chain_read_many")(self._h, gs, ns, fs, cs, C.c_size_t(n), out, present), "chain_read_many")
        res, at = [], 0
        for r in reqs:
            res.append([(out[at + i].id, out[at + i].next, out[at + i].data) if present[at + i] else None
                        for i in range(r[3])])
            at += r[3]
        return res

    def query(self, group: int, node: int) -> abi.ReplicaState:
        st = abi.ReplicaState()
        self._check(self._fn("query")(self._h, C.c_uint32(group), C.c_uint32(node), C.byref(st)), "query")
        return st

    def handle(self, group: int, node: int) -> "ReplicaHandle":
        return ReplicaHandle(self, group, node)

    def chain_read(self, group: int, node: int, first_id: int, n: int) -> List[Optional[Tuple[int, int, int]]]:
        out = (abi.Block * max(n, 1))()
        present = (C.c_uint8 * max(n, 1))()
        self._check(self._fn("chain_read")(self._h, C.c_uint32(group), C.c_uint32(node), C.c_uint64(first_id),
                                           C.c_uint32(n), out, present), "chain_read")
        return [(out[i].id, out[i].next, out[i].data) if present[i] else None for i in range(n)]

    def state_digest(self) -> int:
        v = C.c_uint64(0)
        self._check(self._fn("state_digest")(self._h, C.byref(v)), "state_digest")
        return v.value

    def stream_digest(self) -> Tuple[int, int, int, int]:
        a, b, c, d = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        self._check(self._fn("stream_digest")(self._h, C.byref(a), C.byref(b), C.byref(c), C.byref(d)),
                    "stream_digest")
        return a.value, b.value, c.value, d.value

    def fold_count(self) -> int:
        """Groups the last jr_run* launch applied through the symmetric-group fast path (engine only)."""
        v = C.c_uint64(0)
        self._check(self._fn("fold_count")(self._h, C.byref(v)), "fold_count")
        return v.value

    def fault_count(self) -> int:
        v = C.c_uint64(0)
        self._check(self._fn("fault_count")(self._h, C.byref(v)), "fault_count")
        return v.value

    # -- maintenance ----------------------------------------------------------------
    def compact(self):
        self._check(self._fn("compact")(self._h), "compact")

    def truncate(self, margin: int = 8):
        """jr_truncate (deviation D7): drop every block below min(commit of the live replicas) - margin, per group."""
        self._check(self._fn("truncate")(self._h, C.c_uint32(margin)), "truncate")

    def set_auto_truncate(self, margin: Optional[int] = 8):
        """jr_set_auto_truncate: every fused run ends with jr_truncate(margin); None switches it off."""
        self._check(self._fn("set_auto_truncate")(self._h, C.c_int(0 if margin is None else 1), C.c_uint32(margin or 0)), "set_auto_truncate")

    def node_restart(self, group: int, node: int, now_ms: int, blocks: Sequence[Tuple[int, int, int]], commit: int,
                     commit_key: Optional[bool] = None):
        """jr_node_restart: RaftHandle::new over a persisted chain (chain.rs:117-137)."""
        arr = (abi.Block * max(len(blocks), 1))()
        for i, (bid, nxt, data) in enumerate(blocks):
            arr[i].id, arr[i].next, arr[i].data = bid, nxt, data
        ck = (commit > 0) if commit_key is None else commit_key
        self._check(self._fn("node_restart")(self._h, C.c_uint32(group), C.c_uint32(node), C.c_uint64(now_ms), arr,
                                             C.c_size_t(len(blocks)), C.c_uint64(commit), C.c_int(int(ck))), "node_restart")

    def chain_export_many(self, targets: Sequence[Tuple[int, int]]) -> List[Tuple[int, bool, List[Tuple[int, int, int]]]]:
        """jr_chain_export_many: each (group, node)'s persisted sled tree as (commit, commit_key, [(id, next, token)]),
        every block present in the replica's window, ascending id.  Without the batched call (the oracle): query +
        chain_read per target, and the commit key is taken to exist once something was committed."""
        targets = list(targets)
        n = len(targets)
        if not hasattr(self._lib, self._p + "chain_export_many"):
            out = []
            for g, nd in targets:
                st = self.query(g, nd)
                lo = int(st.chain_floor)
                hi = min(int(st.max_key), lo + self.cfg.chain_capacity - 1)
                blocks = [b for b in self.chain_read(g, nd, lo, hi - lo + 1) if b is not None] if hi >= lo else []
                out.append((int(st.commit), st.commit > 0, blocks))
            return out
        gs = (C.c_uint32 * max(n, 1))(*[t[0] for t in targets])
        ns = (C.c_uint32 * max(n, 1))(*[t[1] for t in targets])
        desc = (abi.PersistedChain * max(n, 1))()
        need = C.c_size_t(0)
        fn = self._fn("chain_export_many")
        st = fn(self._h, gs, ns, C.c_size_t(n), desc, None, C.c_size_t(0), C.byref(need))
        if st != abi.E_CAPACITY:
            self._check(st, "chain_export_many")
        blk = (abi.Block * max(need.value, 1))()
        if need.value:
            self._check(fn(self._h, gs, ns, C.c_size_t(n), desc, blk, need, C.byref(need)), "chain_export_many")
        out = []
        for i in range(n):
            d = desc[i]
            out.append((d.commit, bool(d.commit_key),
                        [(blk[j].id, blk[j].next, blk[j].data) for j in range(d.first_block, d.first_block + d.n_blocks)]))
        return out

    def node_restart_many(self, now_ms: int,
                          chains: Sequence[Tuple[int, int, Optional[Sequence[Tuple[int, int, int]]], int, Optional[bool]]]):
        """jr_node_restart_many: chains = [(group, node, blocks, commit, commit_key)]; blocks None = in place (the replica
        reopens its own table and commit; commit and commit_key are ignored), commit_key None = (commit > 0).  Without
        the batched call (the oracle): one node_restart per entry, in order, in place = from its own export."""
        chains = list(chains)
        if not hasattr(self._lib, self._p + "node_restart_many"):
            for g, nd, blocks, commit, ck in chains:
                if blocks is None:
                    commit, ck, blocks = self.chain_export_many([(g, nd)])[0]
                self.node_restart(g, nd, now_ms, blocks, commit, ck)
            return
        n = len(chains)
        desc = (abi.PersistedChain * max(n, 1))()
        flat: List[Tuple[int, int, int]] = []
        for i, (g, nd, blocks, commit, ck) in enumerate(chains):
            d = desc[i]
            d.group, d.node = g, nd
            if blocks is None:
                d.n_blocks = abi.RESTART_IN_PLACE
                continue
            d.commit, d.first_block, d.n_blocks = commit, len(flat), len(blocks)
            d.commit_key = int((commit > 0) if ck is None else bool(ck))
            flat.extend(blocks)
        arr = (abi.Block * max(len(flat), 1))()
        for i, (bid, nxt, data) in enumerate(flat):
            arr[i].id, arr[i].next, arr[i].data = bid, nxt, data
        self._check(self._fn("node_restart_many")(self._h, C.c_uint64(now_ms), desc, C.c_size_t(n), arr,
                                                  C.c_size_t(len(flat))), "node_restart_many")

    def verify_groups(self, groups: Optional[Sequence[int]] = None) -> Tuple[abi.VerifyReport, List[abi.VerifyFinding]]:
        """jr_verify_groups: check that each group's replicas hold the same committed chain (None = every group).
        Returns (report, findings), findings sorted by (group, node); an empty list means every checked replica agrees.
        Without the batched call (the oracle): the same rules restated over query_many / chain_read_many (verify.py)."""
        if not hasattr(self._lib, self._p + "verify_groups"):
            from .verify import verify_groups
            return verify_groups(self, groups)
        n = 0 if groups is None else len(groups)
        gs = None if groups is None else (C.c_uint32 * max(n, 1))(*groups)
        rep, need = abi.VerifyReport(), C.c_size_t(0)
        fn = self._fn("verify_groups")
        st = fn(self._h, gs, C.c_size_t(n), C.byref(rep), None, C.c_size_t(0), C.byref(need))
        if st == abi.OK:
            return rep, []
        if st != abi.E_CAPACITY:
            self._check(st, "verify_groups")
        buf = (abi.VerifyFinding * need.value)()
        self._check(fn(self._h, gs, C.c_size_t(n), C.byref(rep), buf, need, C.byref(need)), "verify_groups")
        return rep, [buf[i] for i in range(need.value)]

    def export_groups(self, groups: Sequence[int]) -> bytes:
        """jr_group_export: the image of `groups` (sized, then exported).  The groups are detached from this engine."""
        groups = list(groups)
        n = len(groups)
        gs = (C.c_uint32 * max(n, 1))(*groups)
        need = C.c_size_t(0)
        fn = self._fn("group_export")
        st = fn(self._h, gs, C.c_size_t(n), None, C.c_size_t(0), C.byref(need))
        if st != abi.E_CAPACITY:
            self._check(st, "group_export")
        buf = C.create_string_buffer(need.value)
        self._check(fn(self._h, gs, C.c_size_t(n), buf, need, C.byref(need)), "group_export")
        return buf.raw

    def import_groups(self, slots: Sequence[int], image: bytes):
        """jr_group_import: group i of `image` replaces slot slots[i]."""
        slots = list(slots)
        ss = (C.c_uint32 * max(len(slots), 1))(*slots)
        buf = C.create_string_buffer(image, len(image))
        self._check(self._fn("group_import")(self._h, ss, C.c_size_t(len(slots)), buf, C.c_size_t(len(image))), "group_import")

    def save(self) -> bytes:
        """jr_engine_save: checkpoint of everything the engine holds."""
        n = C.c_size_t(0)
        self._check(self._fn("engine_save_size")(self._h, C.byref(n)), "engine_save_size")
        buf = C.create_string_buffer(n.value)
        self._check(self._fn("engine_save")(self._h, buf, n), "engine_save")
        return buf.raw

    def restore(self, blob: bytes):
        buf = C.create_string_buffer(blob, len(blob))
        self._check(self._fn("engine_restore")(self._h, buf, C.c_size_t(len(blob))), "engine_restore")

    def set_alive(self, group: int, node: int, alive: bool):
        self._check(self._fn("set_alive")(self._h, C.c_uint32(group), C.c_uint32(node), C.c_int(int(alive))),
                    "set_alive")

    def kill_leaders(self, salt: int, permille: int) -> int:
        v = C.c_uint64(0)
        self._check(self._fn("kill_leaders")(self._h, C.c_uint64(salt), C.c_uint32(permille), C.byref(v)),
                    "kill_leaders")
        return v.value

    def leader_table(self) -> List[Tuple[int, int, int]]:
        buf = (abi.LeaderEntry * self.n_groups)()
        self._check(self._fn("leader_table")(self._h, buf), "leader_table")
        return [(e.term, e.leader_id, e.commit) for e in buf]

    # -- peer links (F_PEER_LINKS) --------------------------------------------------
    def set_links(self, cuts, groups: Optional[Sequence[int]] = None):
        """jr_set_links: the link matrix of groups[i] becomes cuts[i] (see link_cut / partition).  groups None: `cuts`
        holds one matrix per group.  All or nothing."""
        cuts = list(cuts)
        n = len(cuts)
        if groups is not None and len(groups) != n:
            raise RaftError(abi.E_INVAL, self._p + "set_links", "groups and cuts differ in length")
        cs = (C.c_uint64 * max(n, 1))(*cuts)
        gs = None if groups is None else (C.c_uint32 * max(n, 1))(*groups)
        self._check(self._fn("set_links")(self._h, gs, cs, C.c_size_t(n)), "set_links")

    def links(self, groups: Optional[Sequence[int]] = None) -> List[int]:
        """jr_get_links: the link matrices of `groups` (None: every group)."""
        n = self.n_groups if groups is None else len(groups)
        gs = None if groups is None else (C.c_uint32 * max(n, 1))(*groups)
        out = (C.c_uint64 * max(n, 1))()
        self._check(self._fn("get_links")(self._h, gs, C.c_size_t(n), out), "get_links")
        return list(out[:n])

    def isolate_leaders(self, salt: int, permille: int) -> int:
        """jr_isolate_leaders: kill_leaders' groups for the same salt, each live leader cut off both ways (alive)."""
        v = C.c_uint64(0)
        self._check(self._fn("isolate_leaders")(self._h, C.c_uint64(salt), C.c_uint32(permille), C.byref(v)),
                    "isolate_leaders")
        return v.value

    def link_queues(self, groups: Optional[Sequence[int]] = None):
        """jr_get_link_queues (F_LINK_QUEUES): an (n, 64) uint8 array, [i, 8*(r-1) + (s-1)] = the Messages queued on
        link s -> r of groups[i] (None: every group)."""
        import numpy as np
        n = self.n_groups if groups is None else len(groups)
        gs = None if groups is None else (C.c_uint32 * max(n, 1))(*groups)
        out = (C.c_uint8 * max(64 * n, 1))()
        self._check(self._fn("get_link_queues")(self._h, gs, C.c_size_t(n), out), "get_link_queues")
        return np.frombuffer(bytes(out), np.uint8)[:64 * n].reshape(n, 64).copy()


def link_cut(n_replicas: int, pairs: Iterable[Tuple[int, int]]) -> int:
    """The link matrix that cuts mail from node s to node r for every (s, r) in `pairs` (one direction each)."""
    m = 0
    for s, r in pairs:
        if not (1 <= s <= n_replicas and 1 <= r <= n_replicas) or s == r:
            raise ValueError(f"no link {s} -> {r} in a group of {n_replicas}")
        m |= 1 << (8 * (r - 1) + (s - 1))
    return m


def partition(n_replicas: int, side: Iterable[int]) -> int:
    """The link matrix that cuts every link between the nodes in `side` and the others, in both directions."""
    a = set(side)
    if not a <= set(range(1, n_replicas + 1)):
        raise ValueError(f"nodes of a group of {n_replicas} are 1..{n_replicas}")
    b = set(range(1, n_replicas + 1)) - a
    return link_cut(n_replicas, [(s, r) for s in a for r in b] + [(s, r) for s in b for r in a])


class ReplicaHandle:
    """RaftHandle-style view of one replica (src/raft/mod.rs:437-468)."""

    def __init__(self, api: RaftApi, group: int, node: int):
        self.api, self.group, self.id = api, group, node

    @property
    def state(self) -> abi.ReplicaState:
        return self.api.query(self.group, self.id)

    def is_follower(self) -> bool:
        return self.state.role == abi.ROLE_FOLLOWER

    def is_candidate(self) -> bool:
        return self.state.role == abi.ROLE_CANDIDATE

    def is_leader(self) -> bool:
        return self.state.role == abi.ROLE_LEADER

    def get_head(self) -> int:   # chain.rs:230-232
        return self.state.head

    def get_commit(self) -> int:  # chain.rs:234-236
        return self.state.commit


# ------------------------------------------------------------------------------
_PKG_DIR = os.path.dirname(os.path.abspath(__file__))
ENGINE_LIB_PATH = os.environ.get("JR_ENGINE_LIB") or os.path.join(_PKG_DIR, "csrc", "libjosefine_b200.so")


def _bind(lib: C.CDLL, p: str):
    """Declare argtypes for the functions RaftApi calls (shared by jr_ and jro_)."""
    vp = C.c_void_p
    sig = {
        "step": [vp, C.POINTER(abi.StepArgs)],
        "run": [vp, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32],
        "run_proposals": [vp, C.c_uint64, C.c_uint32, C.c_uint32, C.POINTER(abi.Proposal), C.c_uint32],
        "run_tokens": [vp, C.c_uint64, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint64)],
        "run_token_runs": [vp, C.c_uint64, C.c_uint32, C.c_uint32, C.POINTER(abi.TokenRun)],
        "drain_fsm": [vp, C.POINTER(abi.FsmInstr), C.c_size_t, C.POINTER(C.c_size_t)],
        "query": [vp, C.c_uint32, C.c_uint32, C.POINTER(abi.ReplicaState)],
        "chain_read": [vp, C.c_uint32, C.c_uint32, C.c_uint64, C.c_uint32, C.POINTER(abi.Block),
                       C.POINTER(C.c_uint8)],
        "state_digest": [vp, C.POINTER(C.c_uint64)],
        "stream_digest": [vp] + [C.POINTER(C.c_uint64)] * 4,
        "fault_count": [vp, C.POINTER(C.c_uint64)],
        "fold_count": [vp, C.POINTER(C.c_uint64)],
        "compact": [vp],
        "set_alive": [vp, C.c_uint32, C.c_uint32, C.c_int],
        "kill_leaders": [vp, C.c_uint64, C.c_uint32, C.POINTER(C.c_uint64)],
        "leader_table": [vp, C.POINTER(abi.LeaderEntry)],
        "fsm_records_async": [vp],
        "fsm_records_wait": [vp, C.POINTER(C.POINTER(abi.FsmRecord)), C.POINTER(abi.FsmBatch)],
        "fsm_responses": [vp, C.POINTER(C.POINTER(abi.FsmRecord)), C.POINTER(abi.FsmBatch)],
        "query_many": [vp, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.c_size_t, C.POINTER(abi.ReplicaState)],
        "chain_read_many": [vp, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.POINTER(C.c_uint32),
                            C.c_size_t, C.POINTER(abi.Block), C.POINTER(C.c_uint8)],
        "truncate": [vp, C.c_uint32],
        "node_restart": [vp, C.c_uint32, C.c_uint32, C.c_uint64, C.POINTER(abi.Block), C.c_size_t, C.c_uint64, C.c_int],
        "chain_export_many": [vp, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.c_size_t, C.POINTER(abi.PersistedChain),
                              C.POINTER(abi.Block), C.c_size_t, C.POINTER(C.c_size_t)],
        "node_restart_many": [vp, C.c_uint64, C.POINTER(abi.PersistedChain), C.c_size_t, C.POINTER(abi.Block), C.c_size_t],
        "verify_groups": [vp, C.POINTER(C.c_uint32), C.c_size_t, C.POINTER(abi.VerifyReport), C.POINTER(abi.VerifyFinding),
                          C.c_size_t, C.POINTER(C.c_size_t)],
        "group_export": [vp, C.POINTER(C.c_uint32), C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)],
        "group_import": [vp, C.POINTER(C.c_uint32), C.c_size_t, C.c_void_p, C.c_size_t],
        "engine_save_size": [vp, C.POINTER(C.c_size_t)],
        "engine_save": [vp, C.c_void_p, C.c_size_t],
        "engine_restore": [vp, C.c_void_p, C.c_size_t],
        "set_links": [vp, C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.c_size_t],
        "get_links": [vp, C.POINTER(C.c_uint32), C.c_size_t, C.POINTER(C.c_uint64)],
        "isolate_leaders": [vp, C.c_uint64, C.c_uint32, C.POINTER(C.c_uint64)],
        "get_link_queues": [vp, C.POINTER(C.c_uint32), C.c_size_t, C.POINTER(C.c_uint8)],
    }
    for name, args in sig.items():
        if not hasattr(lib, p + name):   # an older A/B build (JR_ENGINE_LIB): the call site will fail loudly
            continue
        fn = getattr(lib, p + name)
        fn.argtypes = args
        fn.restype = C.c_int
    if hasattr(lib, p + "fsm_expand"):
        fn = getattr(lib, p + "fsm_expand")
        fn.argtypes = [C.POINTER(abi.FsmRecord), C.c_size_t, C.c_uint32, C.c_uint32, C.POINTER(abi.FsmInstr), C.c_size_t,
                       C.POINTER(C.c_size_t)]
        fn.restype = C.c_int
    if hasattr(lib, p + "fsm_fold"):
        fn = getattr(lib, p + "fsm_fold")
        fn.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p]
        fn.restype = C.c_int
    if hasattr(lib, p + "fsm_fold_mt"):
        fn = getattr(lib, p + "fsm_fold_mt")
        fn.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32]
        fn.restype = C.c_int
    et = getattr(lib, p + "election_timeout")
    et.argtypes = [C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32]
    et.restype = C.c_uint32


_engine_lib: Optional[C.CDLL] = None


def expand_records(lib: C.CDLL, records: Sequence[abi.FsmRecord], n_groups: int, n_replicas: int) -> List[abi.FsmInstr]:
    """jr_fsm_expand through ctypes (pure host code: needs no GPU)."""
    n = len(records)
    arr = (abi.FsmRecord * max(n, 1))(*records)
    need = C.c_size_t(0)
    st = lib.jr_fsm_expand(arr, C.c_size_t(n), C.c_uint32(n_groups), C.c_uint32(n_replicas), None, C.c_size_t(0), C.byref(need))
    if st not in (abi.OK, abi.E_CAPACITY):
        raise RaftError(st, "jr_fsm_expand")
    out = (abi.FsmInstr * max(need.value, 1))()
    if need.value:
        st = lib.jr_fsm_expand(arr, C.c_size_t(n), C.c_uint32(n_groups), C.c_uint32(n_replicas), out, need, C.byref(need))
        if st != abi.OK:
            raise RaftError(st, "jr_fsm_expand")
    return [out[i] for i in range(need.value)]


def expand_responses(runs: Sequence[abi.FsmRecord]) -> List[Tuple[int, int, Address, int, int]]:
    """JR_FSMR_RESPONSE runs (as fsm_responses returns them) -> one (group, node, to, request token, block id) per
    ClientResponse, group-major, node ascending, in each replica's apply order (the order fsm.rs:66-76 sends them)."""
    out = []
    for rc in sorted(runs, key=lambda rc: (rc.group, rc.node)):   # stable: FIFO per replica is kept
        to = Address(rc.addr >> 16, rc.addr & 0xFFFF)
        for i in range(rc.count):
            out.append((rc.group, rc.node, to, (rc.tok0 + i * rc.stride) & 0xFFFFFFFFFFFFFFFF, rc.id0 + i))
    return out


def _open_engine_library(path: str) -> C.CDLL:
    lib = C.CDLL(path)
    if hasattr(lib, "jr_is_emulation"):   # tests/emu's host build of the device code: never a product path
        raise RaftError(abi.E_NO_DEVICE, "load_engine_library",
                        f"{path} is the test-only CPU emulation build; there is no CPU fallback")
    return lib


def load_engine_library() -> C.CDLL:
    """Load the CUDA engine.  There is no CPU fallback: a missing library is an error."""
    global _engine_lib
    if _engine_lib is None:
        if not os.path.exists(ENGINE_LIB_PATH):
            raise RaftError(abi.E_NO_DEVICE, "load_engine_library",
                            f"{ENGINE_LIB_PATH} not built; run `python -c 'import __graft_entry__ as g; g.build()'`")
        lib = _open_engine_library(ENGINE_LIB_PATH)
        _bind(lib, "jr_")
        lib.jr_engine_create.argtypes = [C.POINTER(abi.Config), C.POINTER(C.c_void_p)]
        lib.jr_engine_create.restype = C.c_int
        lib.jr_engine_destroy.argtypes = [C.c_void_p]
        lib.jr_engine_destroy.restype = None
        lib.jr_engine_reset.argtypes = [C.c_void_p]
        lib.jr_engine_reset.restype = C.c_int
        lib.jr_engine_set_stream.argtypes = [C.c_void_p, C.c_void_p]
        lib.jr_engine_set_stream.restype = C.c_int
        lib.jr_engine_sync.argtypes = [C.c_void_p]
        lib.jr_engine_sync.restype = C.c_int
        lib.jr_leader_table_device.argtypes = [C.c_void_p, C.c_void_p]
        lib.jr_leader_table_device.restype = C.c_int
        lib.jr_leader_table_async.argtypes = [C.c_void_p, C.POINTER(abi.LeaderEntry)]
        lib.jr_leader_table_async.restype = C.c_int
        if hasattr(lib, "jr_leader_table_wait"):
            lib.jr_leader_table_wait.argtypes = [C.c_void_p]
            lib.jr_leader_table_wait.restype = C.c_int
        lib.jr_config_default.argtypes = [C.POINTER(abi.Config), C.c_uint32, C.c_uint32]
        lib.jr_config_default.restype = None
        lib.jr_last_error.restype = C.c_char_p
        _engine_lib = lib
    return _engine_lib


class RaftEngine(RaftApi):
    """G x R Raft replicas resident in one H100's HBM, stepped by the sm_90a kernels."""

    def __init__(self, cfg: abi.Config):
        lib = load_engine_library()
        h = C.c_void_p()
        st = lib.jr_engine_create(C.byref(cfg), C.byref(h))
        if st != abi.OK:
            raise RaftError(st, "jr_engine_create", (lib.jr_last_error() or b"").decode())
        super().__init__(lib, "jr_", h, cfg)

    @classmethod
    def create(cls, n_groups: int, n_replicas: int, **kw) -> "RaftEngine":
        return cls(abi.default_config(n_groups, n_replicas, **kw))

    def reset(self):
        """Every replica back to a fresh Follower with an empty chain (allocations kept)."""
        self._check(self._lib.jr_engine_reset(self._h), "engine_reset")

    def set_stream(self, cuda_stream: int):
        self._check(self._lib.jr_engine_set_stream(self._h, C.c_void_p(cuda_stream)), "engine_set_stream")

    def sync(self):
        self._check(self._lib.jr_engine_sync(self._h), "engine_sync")

    def leader_table_device(self, dev_ptr: int):
        self._check(self._lib.jr_leader_table_device(self._h, C.c_void_p(dev_ptr)), "leader_table_device")
