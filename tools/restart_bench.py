#!/usr/bin/env python
"""Process restart at full size: how long jr_chain_export_many / jr_node_restart_many take for a broker's worth of replicas,
and what the same restart costs through jr_node_restart one replica at a time.

65,536 groups x 5 replicas, chain_capacity 512, auto-truncate 8 (bench.py's shape), 256 steady ticks first.  Every call
timed here synchronises, so a host clock around it is the call's time.  Prints one line per measurement and a JSON
summary; needs a CUDA device (there is no CPU fallback).
"""
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from josefine_b200 import abi, RaftEngine  # noqa: E402
from tests.stream_cases import _bootstrap  # noqa: E402

G, R, CAP, MARGIN, REPEAT, SINGLES = 65536, 5, 512, 8, 5, 2048


def card() -> str:
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]


def timed(fn, repeat=REPEAT):
    ts = []
    for _ in range(repeat):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts), min(ts), max(ts)


def main():
    eng = RaftEngine.create(G, R, seed=1, chain_capacity=CAP)
    lib, h = eng._lib, eng._h
    _bootstrap(eng, G, R)
    eng.set_auto_truncate(MARGIN)
    for k in range(4):
        eng.run(100 + 6400 * k, 100, 64, 1)
    eng.sync()
    now = 100 + 4 * 6400
    results = {"card": card(), "groups": G, "replicas": R, "chain_capacity": CAP, "auto_truncate": MARGIN}
    print("card:", results["card"])

    def report(name, t, h2d, d2h, **extra):
        med, lo, hi = t
        results[name] = dict(ms_median=med * 1e3, ms_min=lo * 1e3, ms_max=hi * 1e3, h2d_bytes=h2d, d2h_bytes=d2h, **extra)
        print(f"{name:34s} {med * 1e3:9.3f} ms (min {lo * 1e3:.3f}, max {hi * 1e3:.3f})  H2D {h2d / 1e6:8.2f} MB  "
              f"D2H {d2h / 1e6:8.2f} MB  {extra if extra else ''}")

    for label, nodes in (("node2", [2]), ("all", list(range(1, R + 1)))):
        targets = [(g, n) for n in nodes for g in range(G)]      # node-major: each node's requests group-consecutive
        n = len(targets)
        gs = (C.c_uint32 * n)(*[t[0] for t in targets])
        ns = (C.c_uint32 * n)(*[t[1] for t in targets])
        desc = (abi.PersistedChain * n)()
        need = C.c_size_t(0)
        st = lib.jr_chain_export_many(h, gs, ns, n, desc, None, 0, C.byref(need))
        assert st == abi.E_CAPACITY, st
        total = need.value
        blocks = (abi.Block * total)()

        def export():
            assert lib.jr_chain_export_many(h, gs, ns, n, desc, blocks, total, C.byref(need)) == abi.OK

        report(f"export_{label}", timed(export), h2d=n * 8 + n * 32, d2h=n * 32 + total * 24, replicas=n, blocks=total)

        def restart():
            assert lib.jr_node_restart_many(h, C.c_uint64(now), desc, n, blocks, total) == abi.OK

        report(f"restart_{label}_from_export", timed(restart), h2d=n * 32 + total * 24, d2h=G * 4, replicas=n, blocks=total)
        inplace = (abi.PersistedChain * n)()
        for i, (g, nd) in enumerate(targets):
            inplace[i].group, inplace[i].node, inplace[i].n_blocks = g, nd, abi.RESTART_IN_PLACE

        def restart_in_place():
            assert lib.jr_node_restart_many(h, C.c_uint64(now), inplace, n, None, 0) == abi.OK

        report(f"restart_{label}_in_place", timed(restart_in_place), h2d=n * 32, d2h=0, replicas=n)

    # one replica per call, as before the batched call existed: node 2 of the first SINGLES groups, from the export above
    per = []
    for g in range(SINGLES):
        d = desc[(2 - 1) * G + g]
        t0 = time.perf_counter()
        first = C.cast(C.addressof(blocks) + d.first_block * C.sizeof(abi.Block), C.POINTER(abi.Block))
        st = lib.jr_node_restart(h, g, 2, C.c_uint64(now), first, d.n_blocks, d.commit, d.commit_key)
        per.append(time.perf_counter() - t0)
        assert st == abi.OK
    mean = statistics.mean(per)
    results["single_node_restart"] = dict(calls=SINGLES, ms_mean_per_call=mean * 1e3,
                                          extrapolated_node2_ms=mean * G * 1e3, extrapolated_all_ms=mean * G * R * 1e3)
    print(f"jr_node_restart x {SINGLES}: {mean * 1e3:.3f} ms per call; EXTRAPOLATED to {G} replicas: {mean * G:.2f} s, "
          f"to {G * R}: {mean * G * R:.2f} s")
    eng.run(now, 100, 64, 1)
    eng.sync()
    results["faulted_after"] = eng.fault_count()
    print(json.dumps(results))


if __name__ == "__main__":
    main()
