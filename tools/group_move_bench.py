#!/usr/bin/env python
"""Group moves at full size: how long jr_group_export / jr_group_import take for 1, 1,024 and 65,536 groups, listed
group-consecutive and scattered, and how many image bytes a group costs.

65,536 groups x 5 replicas, chain_capacity 512, auto-truncate 8 (bench.py's shape), 256 steady ticks first.  Every call
timed here synchronises, so a host clock around it is the call's time; the median of REPEAT calls is reported.  Each
export is followed by the import of its image into the same slots (a copy that leaves the engine as it was), so every
repeat sees the same state.  GB/s = image bytes over the call's time.  Prints one line per measurement and a JSON
summary; needs a CUDA device (there is no CPU fallback).
"""
import ctypes as C
import json
import os
import random
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from josefine_b200 import abi, RaftEngine  # noqa: E402
from tests.stream_cases import _bootstrap  # noqa: E402

G, R, CAP, MARGIN, REPEAT = 65536, 5, 512, 8, 7


def card() -> str:
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]


def main():
    eng = RaftEngine.create(G, R, seed=1, chain_capacity=CAP)
    lib, h = eng._lib, eng._h
    _bootstrap(eng, G, R)
    eng.set_auto_truncate(MARGIN)
    for k in range(4):
        eng.run(100 + 6400 * k, 100, 64, 1)
    eng.sync()
    digest0 = eng.state_digest()
    results = {"card": card(), "groups": G, "replicas": R, "chain_capacity": CAP, "auto_truncate": MARGIN, "repeat": REPEAT}
    print("card:", results["card"])
    rng = random.Random(7)
    for n in (1, 1024, G):
        for order in ("consecutive", "scattered"):
            groups = list(range(n)) if order == "consecutive" else rng.sample(range(G), n)
            gs = (C.c_uint32 * n)(*groups)
            need = C.c_size_t(0)
            assert lib.jr_group_export(h, gs, n, None, 0, C.byref(need)) == abi.E_CAPACITY
            size = need.value
            buf = C.create_string_buffer(size)
            te, ti = [], []
            for _ in range(REPEAT):
                t0 = time.perf_counter()
                assert lib.jr_group_export(h, gs, n, buf, size, C.byref(need)) == abi.OK
                t1 = time.perf_counter()
                assert lib.jr_group_import(h, gs, n, buf, size) == abi.OK
                t2 = time.perf_counter()
                te.append(t1 - t0)
                ti.append(t2 - t1)
            me, mi = statistics.median(te), statistics.median(ti)
            name = f"{n}_{order}"
            results[name] = dict(image_bytes=size, bytes_per_group=size / n, export_ms=me * 1e3, import_ms=mi * 1e3,
                                 export_gbps=size / me / 1e9, import_gbps=size / mi / 1e9)
            print(f"{name:18s} image {size / 1e6:9.3f} MB ({size / n:8.1f} B/group)  export {me * 1e3:9.3f} ms "
                  f"({size / me / 1e9:6.2f} GB/s)  import {mi * 1e3:9.3f} ms ({size / mi / 1e9:6.2f} GB/s)")
    assert eng.state_digest() == digest0, "export + import into the same slots must leave the engine as it was"
    eng.run(100 + 4 * 6400, 100, 64, 1)
    eng.sync()
    results["faulted_after"] = eng.fault_count()
    results["folded_after"] = eng.fold_count()
    print(json.dumps(results))


if __name__ == "__main__":
    main()
