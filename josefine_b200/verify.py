"""Replica verification restated in Python: the rules of jr_verify_groups (normative in include/josefine_raft_abi.h),
written over query_many / chain_read_many only.

It runs on any RaftApi.  RaftApi.verify_groups falls back to it on an implementation without the batched call (the
oracle), and the tests compare the device's report and findings against it, over the engine's state and the oracle's.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

from . import abi


def _report(values: Sequence[int]) -> abi.VerifyReport:
    rep = abi.VerifyReport()
    for (name, _), v in zip(abi.VerifyReport._fields_, values):
        setattr(rep, name, v)
    return rep


def _finding(group, kind, node, ref, mask, bid, term) -> abi.VerifyFinding:
    f = abi.VerifyFinding()
    f.group, f.kind, f.node, f.ref_node, f.node_mask, f.id, f.term = group, kind, node, ref, mask, bid, term
    return f


def _walk(st: abi.ReplicaState, rows: Dict[int, Tuple[int, int]], W: int):
    """One checked replica's own chain: (kind or None if intact, id, committed chain as a descending id list)."""
    F, c = int(st.chain_floor), int(st.commit)
    if c < F:
        return abi.VERIFY_BELOW_FLOOR, c, []
    if c - F >= W or c not in rows:
        return abi.VERIFY_COMMIT_ABSENT, c, []
    chain, x = [], c
    for _ in range(W):
        row = rows.get(x)
        if row is None or (row[0] >= x and (x or row[0])):   # absent, or a next not below its id (genesis 0 -> 0 excepted)
            return abi.VERIFY_CHAIN_BROKEN, x, []
        chain.append(x)
        if x == 0 or row[0] < F:
            break
        x = row[0]
    return None, c, chain


def verify_groups(api, groups: Optional[Sequence[int]] = None) -> Tuple[abi.VerifyReport, List[abi.VerifyFinding]]:
    """(report, findings) exactly as jr_verify_groups returns them: findings sorted by (group, node), a group's leader
    conflicts (node 0) first, ordered by their lowest leader."""
    from .raft import RaftError
    G, R, W = api.n_groups, api.n_replicas, api.cfg.chain_capacity
    gl = list(range(G)) if groups is None else list(groups)
    if any(not 0 <= g < G for g in gl) or len(set(gl)) != len(gl):
        raise RaftError(abi.E_INVAL, "verify_groups", "a group out of range or named twice")
    gl.sort()
    targets = [(g, n) for g in gl for n in range(1, R + 1)]
    states = dict(zip(targets, api.query_many(targets)))
    checked = {t for t, st in states.items() if st.alive and not st.fault}
    # every block that can be present in a checked replica's window: ids [floor, min(max_key, floor + W - 1)]
    reqs = []
    for t in targets:
        if t in checked:
            lo = int(states[t].chain_floor)
            hi = min(int(states[t].max_key), lo + W - 1)
            if hi >= lo:
                reqs.append((t[0], t[1], lo, hi - lo + 1))
    tables: Dict[Tuple[int, int], Dict[int, Tuple[int, int]]] = {t: {} for t in checked}
    for (g, n, _, _), blocks in zip(reqs, api.chain_read_many(reqs)):
        tables[(g, n)] = {b[0]: (b[1], b[2]) for b in blocks if b is not None}

    counts = [len(gl), len(checked), len(targets) - len(checked), 0, 0, 0, 0, 0]
    findings: List[abi.VerifyFinding] = []
    for g in gl:
        walks = {n: _walk(states[(g, n)], tables[(g, n)], W) for n in range(1, R + 1) if (g, n) in checked}
        intact = [n for n, w in walks.items() if w[0] is None]
        ref = max(intact, key=lambda n: (walks[n][1], -n)) if intact else 0
        out = []
        for n, (kind, bid, chain) in sorted(walks.items()):
            if kind is None and n != ref:
                ref_chain = walks[ref][2]
                if bid not in ref_chain:
                    kind = abi.VERIFY_DIVERGED
                else:
                    rn, rr = tables[(g, n)], tables[(g, ref)]
                    for x in chain:                  # descending: the first difference is the highest
                        if rn[x] != rr.get(x):
                            kind, bid = abi.VERIFY_DIVERGED, x
                            break
            if kind is not None:
                counts[2 + kind] += 1
                out.append(_finding(g, kind, n, ref, 1 << (n - 1), bid, int(states[(g, n)].current_term)))
        leaders: Dict[int, int] = {}
        for n in sorted(walks):
            st = states[(g, n)]
            if st.role == abi.ROLE_LEADER:
                leaders[int(st.current_term)] = leaders.get(int(st.current_term), 0) | (1 << (n - 1))
        conflicts = sorted((mask & -mask, term, mask) for term, mask in leaders.items() if bin(mask).count("1") >= 2)
        counts[7] += len(conflicts)
        findings += [_finding(g, abi.VERIFY_LEADER_CONFLICT, 0, ref, mask, 0, term) for _, term, mask in conflicts]
        findings += out
    return _report(counts), findings
