#!/usr/bin/env python
"""What peer-link cuts cost the steady step (H100 only): bench.py's shape -- 65536 groups x 5 replicas, pre-elected leaders,
auto-truncate, one synthetic proposal per group and tick, 64 ticks per step, Instruction records drained every step -- in
three arms that alternate in one process, round after round:
  off       an engine created without JR_F_PEER_LINKS
  on        with the flag, every matrix zero
  iso10/    with the flag and 1% / 10% of the groups' leaders isolated (jr_isolate_leaders): those groups leave the fold
  iso100    and run through step_kernel
Step time = host clock around one jr_run + the drain of its records, from one device synchronise to the next; the fold count is that of the step's last launch.  Prints one JSON line.

usage: links_bench.py [rounds] [steps per round]"""
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from josefine_b200 import abi, RaftEngine  # noqa: E402
from tests.golden_scenarios import bootstrap  # noqa: E402

G, R, TICKS, DT, MARGIN = 65536, 5, 64, 100, 8


def card():
    out = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm",
                                   "--format=csv,noheader"], text=True).strip()
    return dict(zip(("name", "power_limit", "sm_max_clock"), [x.strip() for x in out.split(",")]))


def engine(flags, isolate_permille):
    e = RaftEngine.create(G, R, seed=1, chain_capacity=512, fsm_units=16, flags=abi.F_CAPTURE_FSM | flags)
    e.step(0, flags=0, inject=bootstrap(G, R))
    e.run(DT, DT, 16, 1)
    e.truncate(MARGIN)
    e.discard_fsm(strict=False)
    e.set_auto_truncate(MARGIN)
    if isolate_permille:
        e.isolate_leaders(12345, isolate_permille)
    return {"eng": e, "now": DT * 17, "ms": [], "fold": []}


def step(a, record):
    e = a["eng"]
    e.sync()
    t0 = time.perf_counter()
    e.run(a["now"], DT, TICKS, 1)
    st = e._lib.jr_fsm_records_async(e._h)
    ptr, batch = C.POINTER(abi.FsmRecord)(), abi.FsmBatch()
    st = st or e._lib.jr_fsm_records_wait(e._h, C.byref(ptr), C.byref(batch))
    assert st in (0, abi.E_CAPACITY), st
    e.sync()
    t1 = time.perf_counter()
    a["now"] += DT * TICKS
    if record:
        a["ms"].append((t1 - t0) * 1e3)
        a["fold"].append(e.fold_count())


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 10
    arms = {"off": engine(0, 0), "on": engine(abi.F_PEER_LINKS, 0), "iso10": engine(abi.F_PEER_LINKS, 10),
            "iso100": engine(abi.F_PEER_LINKS, 100)}
    for a in arms.values():          # warm-up: every shape, and the isolated groups' first launches
        for _ in range(3):
            step(a, False)
    for _ in range(rounds):
        for a in arms.values():
            for _ in range(steps):
                step(a, True)
    out = {"card": card(), "shape": f"{G} groups x {R} replicas, {TICKS} ticks per step", "rounds": rounds,
           "steps_per_round": steps, "arms": {}}
    for name, a in arms.items():
        ms = a["ms"]
        out["arms"][name] = {"ms_per_step_median": statistics.median(ms), "ms_min": min(ms), "ms_max": max(ms),
                             "ms_stdev": statistics.stdev(ms), "fold_count_median": statistics.median(a["fold"]),
                             "groups_cut": sum(1 for m in a["eng"].links() if m) if name != "off" else 0}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
