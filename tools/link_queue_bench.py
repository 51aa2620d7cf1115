#!/usr/bin/env python
"""What link queues cost the steady step (H100 only): bench.py's shape -- 65536 groups x 5 replicas, pre-elected leaders,
auto-truncate, one synthetic proposal per group and tick, 64 ticks per step, Instruction records drained every step -- in
arms that alternate in one process, round after round:
  off        an engine created without JR_F_PEER_LINKS
  links      JR_F_PEER_LINKS only, every matrix zero
  queues     JR_F_PEER_LINKS | JR_F_LINK_QUEUES, no cut
  drop1/10   JR_F_PEER_LINKS only, 1% / 10% of the leaders isolated (jr_isolate_leaders): cut mail is dropped
  queue1/10  both flags, the same groups isolated: cut mail is queued (each link fills up within the first step)
  heal_drop  10% of the leaders isolated for two steps, then healed: the step right after the heal, drop mode
  heal_queue the same in queue mode: the first launch after the heal replays every queue
Step time = host clock around one jr_run + the drain of its records, from one device synchronise to the next; the fold
count is that of the step's last launch.  Prints one JSON line.

usage: link_queue_bench.py [rounds] [steps per round]"""
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
LINKS, QUEUES = abi.F_PEER_LINKS, abi.F_PEER_LINKS | abi.F_LINK_QUEUES


def card():
    out = subprocess.check_output(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm",
                                   "--format=csv,noheader"], text=True).strip()
    return dict(zip(("name", "power_limit", "sm_max_clock"), [x.strip() for x in out.split(",")]))


def engine(flags, isolate_permille=0, heal=False):
    e = RaftEngine.create(G, R, seed=1, chain_capacity=512, fsm_units=16, flags=abi.F_CAPTURE_FSM | flags)
    e.step(0, flags=0, inject=bootstrap(G, R))
    e.run(DT, DT, 16, 1)
    e.truncate(MARGIN)
    e.discard_fsm(strict=False)
    e.set_auto_truncate(MARGIN)
    if isolate_permille and not heal:
        e.isolate_leaders(12345, isolate_permille)
    return {"eng": e, "now": DT * 17, "ms": [], "fold": [], "heal": heal, "salt": 1}


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


def heal_step(a, record):
    """Isolate 10% of the leaders (fresh groups each time), two steps, heal; time the step right after the heal."""
    e = a["eng"]
    a["salt"] += 1
    e.isolate_leaders(a["salt"], 100)
    step(a, False)
    step(a, False)
    a["queued_groups"] = int(e.link_queues().any(axis=1).sum()) if e.cfg.flags & abi.F_LINK_QUEUES else 0
    e.set_links([0] * G)
    step(a, record)
    step(a, False)   # (the old leaders' groups settle before the next round)


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 10
    arms = {"off": engine(0), "links": engine(LINKS), "queues": engine(QUEUES),
            "drop1": engine(LINKS, 10), "queue1": engine(QUEUES, 10), "drop10": engine(LINKS, 100),
            "queue10": engine(QUEUES, 100), "heal_drop": engine(LINKS, heal=True), "heal_queue": engine(QUEUES, heal=True)}
    for a in arms.values():          # warm-up: every shape, and the isolated groups' first launches
        for _ in range(3):
            step(a, False)
    for _ in range(rounds):
        for a in arms.values():
            for _ in range(1 if a["heal"] else steps):
                (heal_step if a["heal"] else step)(a, True)
    out = {"card": card(), "shape": f"{G} groups x {R} replicas, {TICKS} ticks per step", "rounds": rounds,
           "steps_per_round": steps, "arms": {}}
    for name, a in arms.items():
        ms, e = a["ms"], a["eng"]
        out["arms"][name] = {"ms_per_step_median": statistics.median(ms), "ms_min": min(ms), "ms_max": max(ms),
                             "ms_stdev": statistics.stdev(ms) if len(ms) > 1 else 0.0,
                             "fold_count_median": statistics.median(a["fold"]),
                             "groups_cut": sum(1 for m in e.links() if m) if name != "off" else 0}
        if e.cfg.flags & abi.F_LINK_QUEUES:
            out["arms"][name]["groups_queued"] = a.get("queued_groups", int(e.link_queues().any(axis=1).sum()))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
