#!/usr/bin/env python
"""What answering clients from the batched drain costs (JR_F_CLIENT_RESPONSES) at bench.py's headline shape.

65,536 groups x 5 replicas, 64-tick steps of jr_run_token_runs, auto-truncate 8, one drain (jr_fsm_records_async +
jr_fsm_records_wait, and jr_fsm_responses with the flag) per step.  Two engines, flag off and flag on, are stepped
alternately in one process.  CUDA events on the engine stream time the step and the drain's kernels; a host clock times
the drain up to the batch being in host memory.  A torch.profiler pass of its own gives fsm_respond_kernel's time alone, and
a device-to-pinned-host copy of the response runs' bytes on its own gives what their copy costs.
Also reports response runs and device-to-host bytes per step, and the card.  Needs a CUDA device.
"""
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctypes as C  # noqa: E402

import numpy as np  # noqa: E402
import torch  # noqa: E402

from josefine_b200 import abi, RaftEngine  # noqa: E402
from tests.stream_cases import _bootstrap  # noqa: E402

G, R, S, MARGIN, WARMUP, STEPS = 65536, 5, 64, 8, 8, 40


def card() -> str:
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]


class Leg:
    def __init__(self, flags):
        self.eng = RaftEngine.create(G, R, seed=1, flags=flags, chain_capacity=512, fsm_units=16)
        self.resp = bool(flags & abi.F_CLIENT_RESPONSES)
        self.lib, self.h = self.eng._lib, self.eng._h
        self.stream = torch.cuda.Stream()
        self.eng.set_stream(self.stream.cuda_stream)
        _bootstrap(self.eng, G, R)
        self.eng.set_auto_truncate(MARGIN)
        self.eng.run(100, 100, 16, 0)
        self.eng.leader_table()
        self.eng.discard_fsm(strict=False)
        self.now, self.k = 1700, 0
        self.runs = (abi.TokenRun * G)()
        self.tok = np.frombuffer(self.runs, dtype=np.uint64).reshape(G, 2)
        self.tok[:, 1] = 1 << 20
        self.rec = {"step_ms": [], "drain_ms": [], "drain_host_ms": [], "resp_runs": [], "records": [], "d2h_bytes": []}

    def one(self, keep=True):
        self.k += 1
        self.tok[:, 0] = (np.uint64(self.k) << np.uint64(40)) | np.arange(1, G + 1, dtype=np.uint64)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        ev[0].record(self.stream)
        assert self.lib.jr_run_token_runs(self.h, C.c_uint64(self.now), C.c_uint32(100), C.c_uint32(S), self.runs) == 0
        ev[1].record(self.stream)
        t0 = time.perf_counter()
        assert self.lib.jr_fsm_records_async(self.h) == 0
        ev[2].record(self.stream)
        recs, batch = C.POINTER(abi.FsmRecord)(), abi.FsmBatch()
        assert self.lib.jr_fsm_records_wait(self.h, C.byref(recs), C.byref(batch)) == 0
        n_resp = 0
        if self.resp:
            rp, rb = C.POINTER(abi.FsmRecord)(), abi.FsmBatch()
            assert self.lib.jr_fsm_responses(self.h, C.byref(rp), C.byref(rb)) == 0
            n_resp = rb.n_records
        t1 = time.perf_counter()
        self.now += 100 * S
        ev[2].synchronize()
        if keep:
            self.rec["step_ms"].append(ev[0].elapsed_time(ev[1]))
            self.rec["drain_ms"].append(ev[1].elapsed_time(ev[2]))
            self.rec["drain_host_ms"].append((t1 - t0) * 1e3)
            self.rec["resp_runs"].append(n_resp)
            self.rec["records"].append(batch.n_records)
            self.rec["d2h_bytes"].append(32 * (batch.n_records + n_resp))


def main():
    legs = {"off": Leg(abi.F_CAPTURE_FSM), "on": Leg(abi.F_CAPTURE_FSM | abi.F_CLIENT_RESPONSES)}
    for _ in range(WARMUP):
        for leg in legs.values():
            leg.one(keep=False)
    for _ in range(STEPS):                         # alternated: both legs see the same machine state
        for leg in legs.values():
            leg.one()
    out = {"card": card(), "groups": G, "replicas": R, "ticks_per_step": S, "steps": STEPS}
    for name, leg in legs.items():
        out[name] = {k: statistics.median(v) for k, v in leg.rec.items()}
        out[name]["step_ms_min_max"] = [min(leg.rec["step_ms"]), max(leg.rec["step_ms"])]
        out[name]["drain_ms_min_max"] = [min(leg.rec["drain_ms"]), max(leg.rec["drain_ms"])]
    # the respond kernel alone: a profiled pass of its own
    on = legs["on"]
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(10):
            on.one(keep=False)
    torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        if "fsm_" in e.key:
            kern[e.key.split("(")[0]] = {"us_avg": e.device_time_total / max(e.count, 1), "count": e.count}
    out["drain_kernels_on"] = kern
    # what the response runs' copy alone costs: the same bytes, device -> pinned host, on a stream of their own
    nbytes = int(out["on"]["resp_runs"]) * 32
    src = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    dst = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    ts = []
    for _ in range(20):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        dst.copy_(src, non_blocking=True)
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    out["response_copy_ms"] = statistics.median(ts)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
