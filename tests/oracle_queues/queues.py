"""TEST INFRASTRUCTURE ONLY: the oracle (oracle/) with the peer-link calls (tests/oracle_links) and the link queues of
JR_F_LINK_QUEUES (queues.cpp), built from the unchanged sources into a library of its own.

QueueCluster steps every fused call one step at a time, each step preceded by jrq_route_mail: that is where the cuts
and the queues act.  Restarts drop the queues from the restarted node (jrq_drop_sender), as the engine does."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

from josefine_b200 import abi
from josefine_b200.raft import RaftError, _bind
from tests.oracle_links.links import LinkCluster, PyLinkCluster

_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_DIR, "liboracle_queues.so")
_lib = None


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        subprocess.check_call(["make", "-C", _DIR, "-s"])
        lib = C.CDLL(LIB_PATH)
        _bind(lib, "jro_")
        lib.jro_create.argtypes = [C.POINTER(abi.Config), C.c_uint, C.POINTER(C.c_void_p)]
        lib.jro_create.restype = C.c_int
        for name, args in (("jrq_route_mail", [C.c_void_p, C.c_int]), ("jrq_drop_sender", [C.c_void_p, C.c_uint32, C.c_uint32]),
                           ("jrq_reset", [C.c_void_p])):
            getattr(lib, name).argtypes = args
            getattr(lib, name).restype = C.c_int
        lib.jrq_destroy.argtypes = [C.c_void_p]
        lib.jrq_destroy.restype = None
        _lib = lib
    return _lib


class QueueCluster(LinkCluster):
    """LinkCluster of this library: G x R restated nodes whose cut links keep their mail (with F_LINK_QUEUES)."""

    def __init__(self, cfg: abi.Config, n_threads: int = 1):
        lib = load()
        h = C.c_void_p()
        st = lib.jro_create(C.byref(cfg), n_threads, C.byref(h))
        if st != abi.OK:
            raise RaftError(st, "jro_create")
        super(LinkCluster, self).__init__(lib, "jro_", h, cfg)
        self._trunc = None
        self._deliver = True

    @classmethod
    def create(cls, n_groups: int, n_replicas: int, n_threads: int = 1, **kw) -> "QueueCluster":
        return cls(abi.default_config(n_groups, n_replicas, **kw), n_threads)

    def close(self):
        if self._h:
            self._lib.jrq_destroy(self._h)
            self._h = None

    def _route(self):
        self._check(self._lib.jrq_route_mail(self._h, int(self._deliver)), "route_mail")

    def step(self, now_ms, flags=abi.STEP_DELIVER | abi.STEP_TICK, *args, **kw):
        self._deliver = bool(flags & abi.STEP_DELIVER)
        try:
            return super().step(now_ms, flags, *args, **kw)
        finally:
            self._deliver = True

    def node_restart(self, group, node, *args, **kw):
        super().node_restart(group, node, *args, **kw)
        self._check(self._lib.jrq_drop_sender(self._h, group, node), "drop_sender")

    def reset_queues(self):
        """jr_engine_reset's effect on the queues (the oracle has no reset of its own)."""
        self._check(self._lib.jrq_reset(self._h), "reset")


class PyQueueCluster(PyLinkCluster):
    """The independent Python restatement (oracle/restated_raft.py) with the same cuts and queues: in front of every
    delivering step, each sender's previous-step mail is rewritten as jrq_route_mail does."""

    def __init__(self, cfg: abi.Config):
        super().__init__(cfg)
        R = cfg.n_replicas
        self.queues = [[[[] for _s in range(R)] for _r in range(R)] for _g in range(cfg.n_groups)]   # [g][r-1][s-1]

    def link_queues(self):
        R = self.n_replicas
        return [[len(self.queues[g][x // 8][x % 8]) if x // 8 < R and x % 8 < R else 0 for x in range(64)]
                for g in range(self.n_groups)]

    def step(self, now_ms, flags=abi.STEP_DELIVER | abi.STEP_TICK, *args, **kw):
        R = self.n_replicas
        if flags & abi.STEP_DELIVER:
            for g, cut in enumerate(self.cuts):
                Q = self.queues[g]
                if not cut and not any(q for row in Q for q in row):
                    continue
                for n in self.nodes[g]:
                    s, routed = n.s.id, []
                    for r in range(1, R + 1):
                        up = not (cut >> (8 * (r - 1) + (s - 1))) & 1
                        if r != s and up and Q[r - 1][s - 1]:
                            routed += [(abi.ADDR_PEER, r, c) for c in Q[r - 1][s - 1]]
                            Q[r - 1][s - 1] = []
                    for tk, tid, c in n.prev_out:
                        for r in range(1, R + 1):
                            if r == s or not (tk == abi.ADDR_PEERS or (tk == abi.ADDR_PEER and tid == r)):
                                continue
                            if (cut >> (8 * (r - 1) + (s - 1))) & 1:
                                if len(Q[r - 1][s - 1]) < abi.LINK_QUEUE_MSGS:
                                    Q[r - 1][s - 1].append(c)
                            else:
                                routed.append((abi.ADDR_PEER, r, c))
                    n.prev_out = routed
        # the cut mail is routed already: the plain-cut filter of PyLinkCluster must not see it again
        cuts, self.cuts = self.cuts, [0] * self.n_groups
        try:
            return super().step(now_ms, flags, *args, **kw)
        finally:
            self.cuts = cuts
