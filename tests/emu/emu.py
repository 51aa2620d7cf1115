"""TEST INFRASTRUCTURE ONLY: the engine's device code compiled for the host
(tests/emu/cuda_emu.h).  Lets the CPU suite check the CUDA state machine's logic
against the oracle; the shipped library is CUDA-only."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

from josefine_b200 import abi
from josefine_b200.raft import RaftApi, RaftError, _bind

_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_DIR, "libjosefine_emu.so")
_lib = None


def load() -> C.CDLL:
    global _lib
    if _lib is None:
        subprocess.check_call(["make", "-C", _DIR, "-s"])
        lib = C.CDLL(LIB_PATH)
        _bind(lib, "jr_")
        lib.jr_engine_create.argtypes = [C.POINTER(abi.Config), C.POINTER(C.c_void_p)]
        lib.jr_engine_create.restype = C.c_int
        lib.jr_engine_destroy.argtypes = [C.c_void_p]
        lib.jr_engine_destroy.restype = None
        lib.jr_last_error.restype = C.c_char_p
        lib.jr_sym_abort_read.argtypes = [C.c_void_p, C.POINTER(C.c_uint32), C.c_size_t]
        lib.jr_sym_abort_read.restype = C.c_int
        _lib = lib
    return _lib


class EmuEngine(RaftApi):
    def __init__(self, cfg: abi.Config):
        lib = load()
        h = C.c_void_p()
        st = lib.jr_engine_create(C.byref(cfg), C.byref(h))
        if st != abi.OK:
            raise RaftError(st, "jr_engine_create(emu)", (lib.jr_last_error() or b"").decode())
        super().__init__(lib, "jr_", h, cfg)

    @classmethod
    def create(cls, n_groups: int, n_replicas: int, **kw) -> "EmuEngine":
        return cls(abi.default_config(n_groups, n_replicas, **kw))

    def sym_aborts(self) -> dict:
        """jr_sym_abort_read (this build only): {(group, lane): (site, tick)} of the fold's first abort per lane since the
        last call, lane 0 = the leader's side, 1 = the followers'; site is one of SA_* in sym_fold.cuh.  Clears the log."""
        G = self.n_groups
        buf = (C.c_uint32 * (2 * G))()
        self._check(self._lib.jr_sym_abort_read(self._h, buf, C.c_size_t(2 * G)), "sym_abort_read")
        return {(i % G, i // G): (v & 255, v >> 8) for i, v in enumerate(buf) if v}
