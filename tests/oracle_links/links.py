"""TEST INFRASTRUCTURE ONLY: the oracle (oracle/) with the peer-link calls jro_set_links, jro_get_links and
jro_isolate_leaders, built from the unchanged oracle sources plus links.cpp into a library of its own.

LinkCluster steps every fused call one step at a time, each step preceded by jrl_route_mail (links.cpp): that is
where the cuts act.  A fused call's truncation (set_auto_truncate) runs once, after its last step, as in the engine."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from typing import Optional, Sequence, Tuple

from josefine_b200 import abi
from josefine_b200.raft import RaftApi, RaftError, _bind
from oracle.restated_raft import PyCluster

_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_DIR, "liboracle_links.so")
_lib = None


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        subprocess.check_call(["make", "-C", _DIR, "-s"])
        lib = C.CDLL(LIB_PATH)
        _bind(lib, "jro_")
        lib.jro_create.argtypes = [C.POINTER(abi.Config), C.c_uint, C.POINTER(C.c_void_p)]
        lib.jro_create.restype = C.c_int
        lib.jrl_destroy.argtypes = [C.c_void_p]
        lib.jrl_destroy.restype = None
        lib.jrl_route_mail.argtypes = [C.c_void_p]
        lib.jrl_route_mail.restype = C.c_int
        _lib = lib
    return _lib


class LinkCluster(RaftApi):
    """RestatedCluster (oracle/restated.py) of this library: G x R restated nodes whose peer links can be cut."""

    def __init__(self, cfg: abi.Config, n_threads: int = 1):
        lib = load()
        h = C.c_void_p()
        st = lib.jro_create(C.byref(cfg), n_threads, C.byref(h))
        if st != abi.OK:
            raise RaftError(st, "jro_create")
        super().__init__(lib, "jro_", h, cfg)
        self._trunc: Optional[int] = None

    @classmethod
    def create(cls, n_groups: int, n_replicas: int, n_threads: int = 1, **kw) -> "LinkCluster":
        return cls(abi.default_config(n_groups, n_replicas, **kw), n_threads)

    def close(self):
        if self._h:
            self._lib.jrl_destroy(self._h)
            self._h = None

    def _route(self):
        self._check(self._lib.jrl_route_mail(self._h), "route_mail")

    def _end_of_call(self, n_steps: int):
        if self._trunc is not None and n_steps:
            self.truncate(self._trunc)

    def set_auto_truncate(self, margin: Optional[int] = 8):
        self._trunc = margin

    def step(self, now_ms, *args, **kw):
        self._route()
        return super().step(now_ms, *args, **kw)

    def run(self, now0_ms: int, dt_ms: int, n_steps: int, n_synth: int = 0):
        if n_synth > 8:
            raise RaftError(abi.E_INVAL, "jro_run")
        for k in range(n_steps):
            self._route()
            super().run(now0_ms + k * dt_ms, dt_ms, 1, n_synth)
        self._end_of_call(n_steps)

    def run_proposals(self, now0_ms: int, dt_ms: int, proposals, flags: int = 0):
        for k, tick in enumerate(proposals):
            self._route()
            super().run_proposals(now0_ms + k * dt_ms, dt_ms, [tick], flags)
        self._end_of_call(len(proposals))

    def run_tokens(self, now0_ms: int, dt_ms: int, tokens):
        for k, tick in enumerate(tokens):
            self._route()
            super().run_tokens(now0_ms + k * dt_ms, dt_ms, [tick])
        self._end_of_call(len(tokens))

    def run_token_runs(self, now0_ms: int, dt_ms: int, n_steps: int, runs: Sequence[Tuple[int, int]]):
        m = (1 << 64) - 1
        self.run_tokens(now0_ms, dt_ms, [[(b + k * s) & m if b else 0 for b, s in runs] for k in range(n_steps)])


class PyLinkCluster(PyCluster):
    """The independent Python restatement (oracle/restated_raft.py) with the same cuts: in front of every step, each
    sender's previous-step mail is rewritten into what the cut network delivers, as jrl_route_mail does."""

    def __init__(self, cfg: abi.Config):
        super().__init__(cfg)
        self.cuts = [0] * cfg.n_groups

    def set_links(self, cuts, groups=None):
        for g, m in zip(range(self.n_groups) if groups is None else groups, cuts):
            self.cuts[g] = m

    def links(self):
        return list(self.cuts)

    def step(self, now_ms, *args, **kw):
        R = self.n_replicas
        for g, cut in enumerate(self.cuts):
            if not cut:
                continue
            for n in self.nodes[g]:
                s, routed = n.s.id, []
                for tk, tid, c in n.prev_out:
                    for r in range(1, R + 1):
                        up = not (cut >> (8 * (r - 1) + (s - 1))) & 1
                        if r != s and up and (tk == abi.ADDR_PEERS or (tk == abi.ADDR_PEER and tid == r)):
                            routed.append((abi.ADDR_PEER, r, c))
                n.prev_out = routed
        return super().step(now_ms, *args, **kw)
