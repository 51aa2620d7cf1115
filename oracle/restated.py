"""ctypes wrapper of the C++ RESTATEMENT of josefine's src/raft (librestated_raft.so).

TEST INFRASTRUCTURE ONLY -- only tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs may import this.  It is not josefine.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

from josefine_b200 import abi
from josefine_b200.raft import RaftApi, RaftError, _bind

_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_DIR, "librestated_raft.so")
_lib = None


def build(force: bool = False) -> str:
    srcs = [os.path.join(_DIR, f) for f in ("restated_raft.cpp", "restated_cluster.cpp", "restated_raft.hpp")]
    srcs.append(os.path.join(_DIR, "..", "include", "josefine_raft_abi.h"))
    stale = force or not os.path.exists(LIB_PATH) or any(
        os.path.exists(s) and os.path.getmtime(s) > os.path.getmtime(LIB_PATH) for s in srcs)
    if stale:
        subprocess.check_call(["make", "-C", _DIR, "-s"])
    return LIB_PATH


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        build()
        lib = C.CDLL(LIB_PATH)
        _bind(lib, "jro_")
        lib.jro_create.argtypes = [C.POINTER(abi.Config), C.c_uint, C.POINTER(C.c_void_p)]
        lib.jro_create.restype = C.c_int
        lib.jro_destroy.argtypes = [C.c_void_p]
        lib.jro_destroy.restype = None
        lib.jro_shift_ids.argtypes, lib.jro_shift_ids.restype = [C.c_void_p, C.c_uint64], C.c_int
        # direct Chain access for the ported chain.rs tests
        vp, u64 = C.c_void_p, C.c_uint64
        lib.jro_chain_new.argtypes, lib.jro_chain_new.restype = [u64, C.c_int], vp
        lib.jro_chain_free.argtypes, lib.jro_chain_free.restype = [vp], None
        lib.jro_chain_fault.argtypes, lib.jro_chain_fault.restype = [vp], C.c_int
        lib.jro_chain_append.argtypes, lib.jro_chain_append.restype = [vp, u64], u64
        lib.jro_chain_extend.argtypes, lib.jro_chain_extend.restype = [vp, u64, u64, u64], None
        lib.jro_chain_commit.argtypes, lib.jro_chain_commit.restype = [vp, u64], None
        lib.jro_chain_has.argtypes, lib.jro_chain_has.restype = [vp, u64], C.c_int
        lib.jro_chain_compact.argtypes, lib.jro_chain_compact.restype = [vp], None
        lib.jro_chain_head.argtypes, lib.jro_chain_head.restype = [vp], u64
        lib.jro_chain_commit_id.argtypes, lib.jro_chain_commit_id.restype = [vp], u64
        lib.jro_chain_len.argtypes, lib.jro_chain_len.restype = [vp], C.c_size_t
        lib.jro_chain_range_from.argtypes = [vp, u64, C.c_size_t, C.c_size_t, C.POINTER(u64), C.c_size_t]
        lib.jro_chain_range_from.restype = C.c_size_t
        _lib = lib
    return _lib


class RestatedCluster(RaftApi):
    """G x R restated nodes stepped on host cores with the engine's schedule."""

    def __init__(self, cfg: abi.Config, n_threads: int = 1):
        lib = load()
        h = C.c_void_p()
        st = lib.jro_create(C.byref(cfg), n_threads, C.byref(h))
        if st != abi.OK:
            raise RaftError(st, "jro_create")
        super().__init__(lib, "jro_", h, cfg)
        self.n_threads = n_threads

    @classmethod
    def create(cls, n_groups: int, n_replicas: int, n_threads: int = 1, **kw) -> "RestatedCluster":
        return cls(abi.default_config(n_groups, n_replicas, **kw), n_threads)

    def shift_ids(self, k: int):
        """jro_shift_ids (test-only): every group's ids at or above its floor move up by k; needs a quiet cluster."""
        self._check(self._lib.jro_shift_ids(self._h, C.c_uint64(k)), "shift_ids")


class RestatedChain:
    """Direct handle on the restated Chain (chain.rs:99-253) for the ported KATs."""

    def __init__(self, capacity: int = 1 << 20, strict: bool = False):
        self.lib = load()
        self.h = self.lib.jro_chain_new(capacity, int(strict))

    def __del__(self):
        if getattr(self, "h", None):
            self.lib.jro_chain_free(self.h)
            self.h = None

    def append(self, data: int = 0) -> int:
        return self.lib.jro_chain_append(self.h, data)

    def extend(self, id: int, next: int, data: int = 0):
        self.lib.jro_chain_extend(self.h, id, next, data)

    def commit(self, id: int):
        self.lib.jro_chain_commit(self.h, id)

    def has(self, id: int) -> bool:
        return bool(self.lib.jro_chain_has(self.h, id))

    def compact(self):
        self.lib.jro_chain_compact(self.h)

    def get_head(self) -> int:
        return self.lib.jro_chain_head(self.h)

    def get_commit(self) -> int:
        return self.lib.jro_chain_commit_id(self.h)

    def __len__(self) -> int:
        return self.lib.jro_chain_len(self.h)

    @property
    def fault(self) -> int:
        return self.lib.jro_chain_fault(self.h)

    def range_from(self, lo: int, skip: int, take: int):
        buf = (C.c_uint64 * 16)()
        n = self.lib.jro_chain_range_from(self.h, lo, skip, take, buf, 16)
        return [buf[i] for i in range(min(n, 16))]
