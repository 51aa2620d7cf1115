#!/usr/bin/env python
"""Where one bench step's device time goes: CUDA events between the three calls of a step (fused run, truncate, drain)
on the engine's stream, for the headline workload and its variants.  Diagnostic; bench.py holds the reported numbers.

usage: step_breakdown.py [steps] [--kernels]"""
import argparse
import ctypes as C
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402
from josefine_b200 import abi  # noqa: E402


EXPLICIT_TRUNCATE = False


def measure(bn, label, G, R, steps, capture=True, flush=True, **kw):
    torch = bn.torch
    eng = bn.steady_engine(G, R, abi.F_CAPTURE_FSM if capture else 0, auto_truncate=not EXPLICIT_TRUNCATE, **kw)
    lib, h = eng._lib, eng._h
    S = bench.TICKS_PER_STEP
    now = bench.DT_MS * 17
    outstanding = 0
    segs = {"run": [], "truncate": [], "drain": [], "step": []}

    def take():
        ptr, batch = C.POINTER(abi.FsmRecord)(), abi.FsmBatch()
        assert lib.jr_fsm_records_wait(h, C.byref(ptr), C.byref(batch)) == 0

    for i in range(steps + 5):
        if flush:
            bn.flush.fill_(1)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record(bn.stream)
        eng.run(now, bench.DT_MS, S, 1)          # ends with its own truncation (jr_set_auto_truncate) unless --explicit-truncate
        ev[1].record(bn.stream)
        if EXPLICIT_TRUNCATE:
            eng.truncate(bench.TRUNC_MARGIN)
        ev[2].record(bn.stream)
        if capture:
            assert lib.jr_fsm_records_async(h) == 0
            outstanding += 1
        ev[3].record(bn.stream)
        if outstanding == 2:
            take()
            outstanding -= 1
        now += bench.DT_MS * S
        if i >= 5:
            segs["_ev"] = segs.get("_ev", []) + [ev]
    while outstanding:
        take()
        outstanding -= 1
    torch.cuda.synchronize()
    for ev in segs.pop("_ev"):
        segs["run"].append(ev[0].elapsed_time(ev[1]))
        segs["truncate"].append(ev[1].elapsed_time(ev[2]))
        segs["drain"].append(ev[2].elapsed_time(ev[3]))
        segs["step"].append(ev[0].elapsed_time(ev[3]))
    out = {k: round(statistics.mean(v) * 1e3, 1) for k, v in segs.items()}
    print(f"{label:34s} us/step {out}  folded {eng.fold_count()}/{G}  faults {eng.fault_count()}", flush=True)
    del eng
    torch.cuda.empty_cache()


def kernel_times(bn, G, R, steps):
    """Device time per step of every kernel of the headline step (fused run with its pre-pass, drain), from torch.profiler
    in a run of its own: CUDA events between the calls cannot split the fused run into its kernels."""
    from torch.profiler import ProfilerActivity, profile
    torch = bn.torch
    eng = bn.steady_engine(G, R, abi.F_CAPTURE_FSM, auto_truncate=True)
    S = bench.TICKS_PER_STEP
    now = bench.DT_MS * 17

    def step():
        nonlocal now
        bn.flush.fill_(1)
        eng.run(now, bench.DT_MS, S, 1)
        eng.discard_fsm(strict=False)
        now += bench.DT_MS * S

    for _ in range(5):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            step()
        torch.cuda.synchronize()
    rows = [(k.self_device_time_total / steps, k.count / steps, k.key) for k in prof.key_averages() if k.self_device_time_total > 0]
    print(f"kernels of the headline step ({G} groups x {R} replicas, {steps} steps, L2 flushed), us per step:", flush=True)
    for us, n, name in sorted(rows, reverse=True):
        print(f"  {us:9.1f}  x{n:4.1f}  {name[:100]}", flush=True)
    del eng
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("steps", nargs="?", type=int, default=60)
    ap.add_argument("--only", type=int, default=99, help="run only the first N variants")
    ap.add_argument("--explicit-truncate", action="store_true", help="jr_truncate as its own call (the pre-fusion shape)")
    ap.add_argument("--kernels", action="store_true", help="instead: each kernel's device time in the headline step (torch.profiler)")
    a = ap.parse_args()
    global EXPLICIT_TRUNCATE
    EXPLICIT_TRUNCATE = a.explicit_truncate
    bn = bench.Bench(argparse.Namespace())
    G, R = bench.GROUPS_PER_GPU, bench.REPLICAS
    if a.kernels:
        kernel_times(bn, G, R, a.steps)
        return
    variants = [("headline", G, {}), ("headline, no capture", G, {"capture": False}), ("scattered leaders", G, {"scattered": True}),
                ("headline, warm L2 (no flush)", G, {"flush": False}), ("heartbeat every tick", G, {"heartbeat_ms": 99}),
                ("131,072 groups", 2 * G, {}), ("headline, fold off (step_kernel)", G, {"_nofold": True}),
                ("no capture, fold off", G, {"capture": False, "_nofold": True})]
    for label, g, kw in variants[:a.only]:
        if kw.pop("_nofold", False):
            os.environ["JR_NO_FOLD"] = "1"
        measure(bn, label, g, R, a.steps, **kw)


if __name__ == "__main__":
    main()
