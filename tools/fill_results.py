#!/usr/bin/env python
"""Render the measured-results blocks of BASELINE.md and DESIGN.md from one bench.py JSON line.

usage: fill_results.py <bench.json> [<profile_note.txt>]
Rewrites the text between `<!-- results:begin -->` / `<!-- results:end -->` in BASELINE.md and DESIGN.md.
Pure formatting: every number printed comes from the JSON (a bench.py run on an H100, never under a profiler)."""
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def sci(v):
    return "-" if v is None else f"{v:.3g}"


def table(d):
    e2e, dense, plain = d.get("e2e") or {}, d.get("e2e_dense_input") or {}, d.get("e2e_no_output") or {}
    cpu = d.get("cpu_baseline") or {}
    oc, var = d.get("other_configs") or {}, d.get("variants") or {}
    rf = d["roofline"]
    rows = []
    rows.append("| config | what is timed | group-ticks/s | ms per 64-tick step |")
    rows.append("|---|---|---|---|")
    rows.append(f"| #3 65,536x5 steady AE (headline) | device resident: in-kernel proposals, Instruction stream drained to pinned host memory every step | **{sci(d['value'])}** | {d['ms_per_step']:.3f} |")
    if e2e:
        rows.append(f"| #3 | end to end, run-length input + Instruction stream folded on the host (`e2e`) | **{sci(e2e['value'])}** | {e2e['ms_per_step']:.3f} (H2D {e2e['h2d_bytes_per_step'] / 1e6:.1f} MB, D2H {e2e['d2h_bytes_per_step'] / 1e6:.1f} MB per step) |")
    if dense:
        rows.append(f"| #3 | end to end, dense 8-byte tokens in + Instruction stream out | {sci(dense['value'])} | {dense['ms_per_step']:.3f} (H2D {dense['h2d_bytes_per_step'] / 1e6:.1f} MB) |")
    if plain:
        rows.append(f"| #3 | end to end WITHOUT the Instruction stream (round 1's leg: dense tokens in, leader table out) | {sci(plain['value'])} | {plain['ms_per_step']:.3f} |")
    for key, label in (("scattered_leaders", "#3 with leaders scattered over the nodes"), ("heartbeat_every_tick", "#3 with a heartbeat every tick (heartbeat_ms = 99)")):
        if key in var:
            rows.append(f"| {label} | device resident | {sci(var[key]['value'])} | {var[key]['ms_per_step']:.3f} |")
    if "config2" in oc:
        c = oc["config2"]
        rows.append(f"| #2 1,024x3 cold start + 64 proposals, 256 ticks | device resident, whole trace | {sci(c['value'])} | {c['ms_per_trace']:.3f} per 256-tick trace ({c['groups_with_leader']} groups elected a leader) |")
    if "config4_shard" in oc:
        c = oc["config4_shard"]
        rows.append(f"| #4 shard: 131,072x5 per GPU x {d['n_gpus']} GPU(s) | device resident | {sci(c['value'])} | {c['ms_per_step']:.3f} |")
    if "config5" in oc:
        c = oc["config5"]
        ck = c["compact_kernel"]
        rows.append(f"| #5 65,536x7, 10% leaders silenced / 100 ticks, compact / 256 ticks | device resident | {sci(c['value'])} | {c['ms_per_step']:.3f}; `compact_kernel` {ck['ms'] if ck['ms'] is None else round(ck['ms'] * 1e3)} us over {ck['bytes'] / 1e6:.1f} MB ({sci(ck['gbs'])} GB/s); {c['groups_with_live_leader_at_end']} groups still led at the end |")
    if cpu:
        rows.append(f"| #3, C++ restatement of src/raft on the host (NOT josefine) | same step, {cpu['cores']} threads / 1 thread | {sci(cpu['value'])} / {sci(cpu.get('value_1_thread'))} | - |")
    out = "\n".join(rows)
    out += (f"\n\nRoofline of the headline line (`roofline` in the JSON): {rf['algorithmic_bytes_per_group_tick']:.0f} B per group-tick in the reference's "
            f"widths -> {rf['achieved']:.0f} GB/s = **{rf['frac']:.2f}** of the HBM peak ({rf['peak']:.0f} GB/s, {rf['peak_source']}); in this engine's wider "
            f"layout {rf['layout_bytes_per_group_tick']:.0f} B -> {rf['frac_layout']:.2f}; real DRAM traffic of the dominant kernel "
            f"{'n/a' if rf.get('frac_dram') is None else format(rf['frac_dram'], '.2f')} of peak.  Parity in the same run: "
            + ", ".join(f"{p['config']}: {'bit-exact' if p['bit_exact'] else 'MISMATCH'}" for p in d.get("parity") or []) + ".")
    if d.get("gpu"):
        out += f"  Card: {d['gpu']['name']}, power limit {d['gpu']['power_limit']}, max SM clock {d['gpu']['sm_max_clock']}."
    if d.get("clocks"):
        out += f"  Clocks during the timed region: {d['clocks']['sm_mhz']} / {d['clocks']['sm_max_mhz']} MHz, reasons {d['clocks']['reasons']}."
    return out


def main():
    d = json.loads([l for l in open(sys.argv[1]) if l.startswith("{")][-1])
    block = table(d)
    for name in ("BASELINE.md", "DESIGN.md"):
        p = os.path.join(ROOT, name)
        s = open(p).read()
        new = re.sub(r"<!-- results:begin -->.*?<!-- results:end -->", lambda _m: "<!-- results:begin -->\n" + block + "\n<!-- results:end -->", s, flags=re.S)
        new = re.sub(r"<!-- refbytes -->.*?<!-- /refbytes -->", lambda _m: f"<!-- refbytes -->{d['roofline']['algorithmic_bytes_per_group_tick']:.0f}<!-- /refbytes -->", new, flags=re.S)
        if new == s and "<!-- results:begin -->" not in s:
            print(f"{name}: no results block")
        open(p, "w").write(new)
    print(block)


if __name__ == "__main__":
    main()
