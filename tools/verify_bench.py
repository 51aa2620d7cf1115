#!/usr/bin/env python
"""What jr_verify_groups costs at the headline shape: 65,536 groups x 5 replicas, chain_capacity 512.

Two states, each after its own steady run:
  truncated    auto-truncate 8, 256 ticks: about a dozen committed blocks per replica inside the window
  full_window  no truncation, 448 ticks: every walk covers about 450 blocks of the 512-id window
For each: the host-clock time of the call (it synchronises), median of REPEAT calls, and in a separate torch.profiler
pass the device time of its kernels per call.  The card's name and power limit are read in the same run.  Needs a CUDA
device (there is no CPU fallback).
"""
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from josefine_b200 import RaftEngine  # noqa: E402
from tests.stream_cases import _bootstrap  # noqa: E402

G, R, CAP, REPEAT, PROFILED = 65536, 5, 512, 21, 10


def card() -> str:
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]


def engine(margin, ticks):
    eng = RaftEngine.create(G, R, seed=1, chain_capacity=CAP)
    _bootstrap(eng, G, R)
    eng.set_auto_truncate(margin)
    eng.run(100, 100, 8, 1)
    eng.leader_table()
    runs = [(1 << 40 | (g + 1), 1 << 20) for g in range(G)]
    for k in range(ticks // 64):
        eng.run_token_runs(900 + 6400 * k, 100, 64, runs)
    eng.sync()
    assert eng.fault_count() == 0
    return eng


def main():
    out = {"card": card(), "groups": G, "replicas": R, "chain_capacity": CAP, "calls": REPEAT}
    print("card:", out["card"])
    for name, margin, ticks in (("truncated", 8, 256), ("full_window", None, 448)):
        eng = engine(margin, ticks)
        st = eng.query(0, 1)
        rep, findings = eng.verify_groups()                    # warm-up: loads the kernels, allocates the scratch
        assert not findings and rep.replicas_checked == G * R, (rep.as_tuple(), len(findings))
        ts = []
        for _ in range(REPEAT):
            t0 = time.perf_counter()
            eng.verify_groups()
            ts.append(time.perf_counter() - t0)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(PROFILED):
                eng.verify_groups()
        torch.cuda.synchronize()
        kern = {e.key.split("(")[0]: e.device_time_total / PROFILED for e in prof.key_averages() if "verify_" in e.key}
        rows = int(st.commit) - int(st.chain_floor) + 1
        out[name] = dict(commit=int(st.commit), floor=int(st.chain_floor), call_ms_median=statistics.median(ts) * 1e3,
                         call_ms_min=min(ts) * 1e3, call_ms_max=max(ts) * 1e3, kernel_us_per_call=kern,
                         kernel_us_total=sum(kern.values()),
                         # rows read: every replica's own walk (4 B next a row), then each non-reference replica's
                         # compare walk (next and token of its row and of the reference's: 24 B a row)
                         table_bytes_walked=G * R * rows * 4 + G * (R - 1) * rows * 24)
        print(name, json.dumps(out[name]))
        eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
