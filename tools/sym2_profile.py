#!/usr/bin/env python
"""Warp-cycle attribution of the symmetric-group fold (sym2_kernel) with the JR_PROFILE build
(josefine_b200/csrc/ab/lib_prof.so, `python __graft_entry__.py --profile-build`): where a leader warp's and a follower
warp's cycles go per tick, at the headline shape (65,536 groups x 5 replicas, 64 ticks per launch).  Lane 0 of every
warp adds clock64() deltas to per-(role, phase) counters; every cycle of a tick lands in exactly one phase, so a lane's
phases add up to its tick and the barrier phase says which lane waits for the other.  The profile build is for
attribution only: the clock reads themselves cost cycles, so its totals are not the benchmark's.

usage: sym2_profile.py [launches]"""
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("JR_ENGINE_LIB", os.path.join(ROOT, "josefine_b200", "csrc", "ab", "lib_prof.so"))
if not os.path.exists(os.environ["JR_ENGINE_LIB"]):
    raise SystemExit("build it first (here, no GPU needed): python __graft_entry__.py --profile-build")
import bench  # noqa: E402
from josefine_b200 import abi, RaftEngine  # noqa: E402

# the slots of sym_fold.cuh (SP_*)
TICK = {0: "mail read (+ proposal)", 1: "AppendResponse (leader_commit loop)", 2: "client_request", 3: "NOTIFY encoder pushes",
        4: "APPLY encoder pushes", 5: "heartbeat / mail write", 7: "heartbeat + apply range", 8: "replicate scan (fetch_sent)",
        9: "follower_extend (row stores)", 6: "barrier wait"}
LAUNCH = {10: "entry record load", 11: "cache fill + encoder init", 12: "sym_leave", 13: "fused truncation"}
LEADER, FOLLOWER = 2, 0


def main():
    launches = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    G, R, S = bench.GROUPS_PER_GPU, bench.REPLICAS, bench.TICKS_PER_STEP
    e = RaftEngine.create(G, R, seed=bench.SEED, chain_capacity=bench.CHAIN_WINDOW, flags=abi.F_CAPTURE_FSM,
                          fsm_units=bench.FSM_UNITS, mailbox_units=64)   # the bench's engine (steady_engine)
    e.step(0, flags=0, inject=bench.bootstrap_inject(G, R))
    e.run(100, 100, 16, 1)
    e.truncate(bench.TRUNC_MARGIN)
    e.discard_fsm(strict=False)
    e.set_auto_truncate(bench.TRUNC_MARGIN)
    now = 1700
    for _ in range(3):                           # into the steady state, where every group folds
        e.run(now, 100, S, 1)
        e.discard_fsm(strict=False)
        now += 100 * S
    buf = (C.c_uint64 * 96)()
    e._lib.jr_profile_read.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
    e._lib.jr_profile_read(e._h, buf)           # clear
    for _ in range(launches):
        e.run(now, 100, S, 1)
        e.discard_fsm(strict=False)
        now += 100 * S
    e._lib.jr_profile_read(e._h, buf)
    print(f"sym2_kernel<{R}> phase profile: {G} groups x {R} replicas, {launches} launches of {S} ticks, "
          f"folded {e.fold_count()}/{G}, faults {e.fault_count()}")
    for role, rn in ((LEADER, "LEADER warp"), (FOLLOWER, "FOLLOWER warp")):
        cyc = lambda s: buf[(role * 16 + s) * 2]
        cnt = lambda s: buf[(role * 16 + s) * 2 + 1]
        ticks = cnt(6) or 1                      # one barrier per warp-tick
        total = sum(cyc(s) for s in TICK)
        print(f"== {rn}: cycles per warp-tick ({ticks} warp-ticks), {total / ticks:.0f} in all")
        for s, name in TICK.items():
            if cnt(s):
                print(f"  {name:38s} {cyc(s) / ticks:8.0f}  {100 * cyc(s) / total:5.1f}%   x{cnt(s) / ticks:5.2f} per tick")
        warps = cnt(10) or 1
        print(f"   once per launch, cycles per warp ({warps} warp-launches):")
        for s, name in LAUNCH.items():
            if cnt(s):
                print(f"  {name:38s} {cyc(s) / warps:8.0f}")
    # the followers' write-back row cache (SP_DROPPED / SP_WRITTEN): dirty rows per group-launch, [0] evicted by an
    # append, [1] left at the exit.  Nearly every eviction should be a drop; many write-backs mean the cache is too small
    # for the truncation margin.
    gl = G * launches
    row = lambda s: (buf[(FOLLOWER * 16 + s) * 2] / gl, buf[(FOLLOWER * 16 + s) * 2 + 1] / gl)
    (de, dx), (we, wx) = row(14), row(15)
    print(f"== followers' dirty rows per group-launch: on eviction {de:.2f} dropped / {we:.2f} written back; "
          f"at the exit {dx:.2f} dropped / {wx:.2f} written back")


if __name__ == "__main__":
    main()
