"""TEST INFRASTRUCTURE ONLY: the oracle (oracle/) with jro_group_move, the restatement of jr_group_export +
jr_group_import, built from the unchanged oracle sources plus group_move.cpp into a library of its own."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

from josefine_b200 import abi
from josefine_b200.raft import RaftApi, RaftError, _bind

_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_DIR, "liboracle_move.so")
_lib = None


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        subprocess.check_call(["make", "-C", _DIR, "-s"])
        lib = C.CDLL(LIB_PATH)
        _bind(lib, "jro_")
        lib.jro_create.argtypes = [C.POINTER(abi.Config), C.c_uint, C.POINTER(C.c_void_p)]
        lib.jro_create.restype = C.c_int
        lib.jro_destroy.argtypes = [C.c_void_p]
        lib.jro_destroy.restype = None
        lib.jro_group_move.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32), C.c_size_t]
        lib.jro_group_move.restype = C.c_int
        _lib = lib
    return _lib


class MovableCluster(RaftApi):
    """RestatedCluster (oracle/restated.py) of this library: G x R restated nodes whose groups can move."""

    def __init__(self, cfg: abi.Config, n_threads: int = 1):
        lib = load()
        h = C.c_void_p()
        st = lib.jro_create(C.byref(cfg), n_threads, C.byref(h))
        if st != abi.OK:
            raise RaftError(st, "jro_create")
        super().__init__(lib, "jro_", h, cfg)

    @classmethod
    def create(cls, n_groups: int, n_replicas: int, n_threads: int = 1, **kw) -> "MovableCluster":
        return cls(abi.default_config(n_groups, n_replicas, **kw), n_threads)

    def group_move(self, dst: "MovableCluster", groups, slots):
        """jro_group_move: jr_group_export of `groups` here + jr_group_import into `slots` of dst."""
        groups, slots = list(groups), list(slots)
        if len(slots) != len(groups):
            raise RaftError(abi.E_INVAL, "jro_group_move", "groups and slots differ in length")
        n = len(groups)
        gs = (C.c_uint32 * max(n, 1))(*groups)
        ss = (C.c_uint32 * max(n, 1))(*slots)
        self._check(self._lib.jro_group_move(self._h, dst._h, gs, ss, C.c_size_t(n)), "group_move")
