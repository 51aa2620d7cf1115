"""bench.py's JSON contract, as far as it can be checked without a GPU: the reference arm
(the C++ restatement on host cores) prints ONE JSON line with the keys the driver reads."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_the_contract_line():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1",
                          "--warmup", "1", "--groups", "2048"], capture_output=True, text=True, timeout=280, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    line = [l for l in out.stdout.splitlines() if l.startswith("{")][-1]
    d = json.loads(line)
    for key in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better",
                "scaling", "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e"):
        assert key in d, key
    assert d["impl"] == "reference" and d["metric"].startswith("Raft-group ticks/sec") and d["unit"] == "group-ticks/s"
    assert d["value"] > 1e4 and d["higher_is_better"] is True and d["vs_baseline"] is None
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["value"] == d["value"]
    assert d["e2e"] == {"value": d["value"], "unit": d["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert "restatement" in d["config"]["comparator"] and "workload" in d["config"]


def test_reference_arm_nonzero_rank_exits_quietly():
    env = dict(os.environ, RANK="1", WORLD_SIZE="2")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2",
                          "--steps", "1", "--warmup", "1"], capture_output=True, text=True, timeout=120, cwd=ROOT, env=env)
    assert out.returncode == 0 and out.stdout.strip() == ""


def _bench():
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import bench
    return bench


def test_dump_record_columns_follow_the_abi_header():
    """--dump-outputs decodes jr_fsm_record as JR_FSMR_KIND / NODE / COUNT and splits u64 fields into exact u32 halves."""
    import ctypes as C

    import numpy as np
    from josefine_b200 import abi
    bench = _bench()
    recs = (abi.FsmRecord * 2)()
    r = recs[1]
    r.group, r.hdr, r.id0, r.addr = 70000, 2 | (4 << 2) | (300 << 8), 123, 0b11110
    r.tok0, r.stride = (0xFFFFFFFF << 32) | 7, (1 << 32) | 0xFFFFFFFF
    got = bench.record_arrays(C.cast(recs, C.POINTER(abi.FsmRecord)), 2)
    assert got.dtype == np.float64 and got.shape == (2, len(bench.RECORD_COLUMNS))
    assert list(got[0]) == [0, 0, 1, 0, 0, 0, 0, 0, 0, 0]                     # an all-zero record is node 1
    row = dict(zip(bench.RECORD_COLUMNS, got[1]))
    assert row == {"group": 70000, "kind": 2, "node": 5, "count": 300, "id0": 123, "addr": 0b11110,
                   "tok0_lo": 7, "tok0_hi": 0xFFFFFFFF, "stride_lo": 0xFFFFFFFF, "stride_hi": 1}
    assert row["kind"] == abi.FsmRecord.from_buffer_copy(recs[1]).kind and row["node"] == abi.FsmRecord.from_buffer_copy(recs[1]).node


def test_dump_outputs_samples_large_batches_the_same_way_every_time(tmp_path, monkeypatch):
    import numpy as np
    bench = _bench()
    monkeypatch.setattr(bench, "DUMP_RECORD_ROWS", 100)
    records = np.arange(1000 * len(bench.RECORD_COLUMNS), dtype=np.float64).reshape(1000, -1)
    table = [(1, 1, 5), (2, 3, 9)]
    for d in ("a", "b"):
        bench.dump_outputs(str(tmp_path / d), table, records)
    a, b = (np.load(tmp_path / d / "fsm_records.npy") for d in ("a", "b"))
    assert a.shape == (100, len(bench.RECORD_COLUMNS)) and np.array_equal(a, b)
    assert (np.diff(a[:, 0]) > 0).all()                                       # rows keep the drain's order
    assert np.array_equal(np.load(tmp_path / "a" / "leader_table.npy"), np.array(table, dtype=np.float64))
    bench.dump_outputs(str(tmp_path / "small"), table, records[:50])         # within the limit: every row
    assert np.array_equal(np.load(tmp_path / "small" / "fsm_records.npy"), records[:50])
