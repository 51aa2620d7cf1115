"""Bulk chain export and bulk node restart (jr_chain_export_many / jr_node_restart_many): a process's worth of replicas
saved and reopened in one call each.  Checked on the device code (CPU emulation) and on the GPU against the oracle's
loop of single restarts (chain.rs:117-137), against the engine's own export + restart, around the symmetric-group
fold, and at full size."""
import ctypes as C
import os
import subprocess

import pytest

from josefine_b200 import abi, Command, persist
from tests import parity
from tests.stream_cases import _bootstrap
from tests.test_sym_fold import same, trio

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _oracle(g, r, **kw):
    from oracle.restated import RestatedCluster
    return RestatedCluster.create(g, r, n_threads=16 if g >= 1024 else 1, **kw)


def _emu(g, r, **kw):
    from tests.emu.emu import EmuEngine
    return EmuEngine.create(g, r, **kw)


def _gpu(g, r, **kw):
    from josefine_b200 import RaftEngine
    return RaftEngine.create(g, r, **kw)


def window(api, g, n):
    """(commit, blocks present in [floor, max_key]) through query + chain_read."""
    st = api.query(g, n)
    lo, hi = int(st.chain_floor), int(st.max_key)
    return int(st.commit), ([b for b in api.chain_read(g, n, lo, hi - lo + 1) if b is not None] if hi >= lo else [])


def _history(make, G, R, seed, strict=False):
    """Oracle / engine pair after elections, proposals, truncation, compaction and a dead branch on a follower."""
    cfg = dict(seed=seed, chain_capacity=32, fsm_units=64,
               flags=parity.FULL | (abi.F_SLED_COMMIT_KEY_STRICT if strict else 0))
    p = parity.Pair(_oracle, make, G, R, check_states_every=0, chain_ids=48, **cfg)
    parity.bootstrap_leaders(p, now=0)
    now = 0
    for _ in range(12):
        now += 100
        p.step(now, n_synth=1)
    p.both("truncate", 3)
    p.both("compact")
    # node 2 of group 0 extends a block whose parent lies below its head: a branch the leader's next blocks overwrite
    st = p.b.query(0, 2)
    now += 100
    p.step(now, flags=0, inject=[Command.append_entries(0, 2, term=int(st.current_term), leader_id=1,
                                                        blocks=[(int(st.head) + 2, int(st.head) - 1, 777)])])
    for _ in range(6):
        now += 100
        p.step(now, n_synth=1)
    p.both("truncate", 4)
    if not strict:   # (strict: the commit key's range panic, D6, stops replicas before the window moves)
        assert any(int(p.b.query(g, 1).chain_floor) > 0 for g in range(G))
    return p, now, cfg


def case_export_and_restart(make, R, strict=False, G=6, seed=3):
    p, now, _ = _history(make, G, R, seed, strict)
    eng, ora = p.b, p.a
    targets = [(g, n) for g in range(G) for n in range(1, R + 1)]
    exp = eng.chain_export_many(targets + targets[:3])            # targets may repeat
    assert exp[-3:] == exp[:3]
    exp = exp[:len(targets)]
    for (g, n), (commit, ck, blocks) in zip(targets, exp):
        assert (commit, blocks) == window(eng, g, n), (g, n)
    assert [(c, b) for c, _, b in exp] == [(c, b) for c, _, b in ora.chain_export_many(targets)]
    for api in (eng, ora):
        assert persist.export_many(api, targets) == {t: persist.chain_records(api, *t) for t in targets}
    # node 2 of every group and node R of every other group, from the export: the oracle's single restarts in order
    by = dict(zip(targets, exp))
    pick = [(g, 2) for g in range(G)] + [(g, R) for g in range(0, G, 2)]
    chains = [(g, n, by[(g, n)][2], by[(g, n)][0], by[(g, n)][1]) for g, n in pick]
    now += 50
    eng.node_restart_many(now, chains)
    for g, n, blocks, commit, ck in chains:
        ora.node_restart(g, n, now, blocks, commit, ck)
    parity.compare_states(ora, eng, chain_ids=64, where="[restarted]")
    parity.compare_digests(ora, eng, "[restarted]")
    for _ in range(100):
        now += 100
        p.step(now, n_synth=1)
    p.finish()


def case_in_place_equals_export(make, R, G=6, seed=4):
    """JR_RESTART_IN_PLACE == export + restart from the export, on a clone of the same engine -- and == the oracle."""
    p, now, cfg = _history(make, G, R, seed)
    a, ora = p.b, p.a
    b = make(G, R, **cfg)
    b.restore(a.save())
    pick = [(g, n) for g in range(G) for n in range(1, R + 1) if (g + n) % 2 == 0]
    a.node_restart_many(now, [(g, n, None, 0, None) for g, n in pick])
    exp = b.chain_export_many(pick)
    b.node_restart_many(now, [(g, n, bl, c, ck) for (g, n), (c, ck, bl) in zip(pick, exp)])
    assert a.state_digest() == b.state_digest()
    parity.compare_states(a, b, chain_ids=64)
    assert a.save() == b.save()
    ora.node_restart_many(now, [(g, n, None, 0, None) for g, n in pick])
    parity.compare_states(ora, a, chain_ids=64, where="[in place]")
    parity.compare_digests(ora, a, "[in place]")
    for _ in range(20):
        now += 100
        p.step(now, n_synth=1)
    p.finish()


def case_commit_without_key(make):
    """A tree restarted with a commit value but no "commit" key (D6) exports exactly that, from host data and in place."""
    api = make(2, 3, seed=1, chain_capacity=32)
    _bootstrap(api, 2, 3)
    api.run(100, 100, 10, 1)
    (commit, ck, blocks), = api.chain_export_many([(1, 2)])
    assert commit > 0 and ck and blocks
    api.node_restart_many(5000, [(1, 2, blocks, commit, False)])
    assert api.chain_export_many([(1, 2)]) == [(commit, False, blocks)]
    api.node_restart_many(5100, [(1, 2, None, 0, None)])
    assert api.chain_export_many([(1, 2)]) == [(commit, False, blocks)]
    st = api.query(1, 2)
    assert (st.head, st.commit, st.id_gen, st.election_time_ms) == (commit, commit, commit, 5100)


def _restart_raw(api, chains, blocks, n_blocks=None):
    desc = (abi.PersistedChain * max(len(chains), 1))()
    for i, c in enumerate(chains):
        for k, v in c.items():
            setattr(desc[i], k, v)
    arr = (abi.Block * max(len(blocks), 1))()
    for i, (bid, nxt, tok) in enumerate(blocks):
        arr[i].id, arr[i].next, arr[i].data = bid, nxt, tok
    n_blocks = len(blocks) if n_blocks is None else n_blocks
    return api._fn("node_restart_many")(api._h, C.c_uint64(9000), desc, C.c_size_t(len(chains)), arr, C.c_size_t(n_blocks))


def case_rejections(make):
    G, R, cap = 4, 3, 16
    api = make(G, R, seed=2, chain_capacity=cap)
    _bootstrap(api, G, R)
    api.run(100, 100, 20, 1)
    api.truncate(2)
    floor = int(api.query(1, 2).chain_floor)
    (commit, _, good), = api.chain_export_many([(1, 2)])
    assert floor > 0 and len(good) >= 3 and good[0][0] >= floor
    ok = dict(group=1, node=2, commit=commit, first_block=0, n_blocks=len(good), commit_key=1)
    inplace = dict(group=0, node=1, n_blocks=abi.RESTART_IN_PLACE)
    swapped = [good[1], good[0]] + good[2:]
    repeated = [good[0], good[0]] + good[2:]
    bad = [
        ([dict(ok, group=G)], good),
        ([dict(ok, node=0)], good),
        ([dict(ok, node=R + 1)], good),
        ([ok, dict(ok, n_blocks=abi.RESTART_IN_PLACE)], good),          # one replica twice
        ([dict(inplace), dict(inplace, first_block=5)], []),             # ... also in place
        ([dict(ok, first_block=1)], good),                               # slice runs past the array
        ([ok], good, len(good) - 1),                                     # ... past the call's n_blocks
        ([dict(ok, n_blocks=cap + 1)], [(floor + k, floor + k - 1, 0) for k in range(cap + 1)]),
        ([ok], swapped),                                                 # not ascending
        ([ok], repeated),                                                # not strictly ascending
        ([ok], [(floor - 1, floor - 2, 0)] + good[1:]),                  # below the floor
        ([ok], good[:-1] + [(floor + cap, floor, 0)]),                   # past the window
        ([ok], good[:-1] + [(good[-1][0], 0xFFFFFFFF, 0)]),              # next = 2^32-1
        ([dict(ok, commit=0xFFFFFFFF)], good),                           # commit = 2^32-1
        ([inplace, dict(ok, group=G)], good),                            # a good request does not go through alone
    ]
    before = api.state_digest()
    for case in bad:
        assert _restart_raw(api, *case) == abi.E_INVAL, case
        assert api.state_digest() == before, case
    assert _restart_raw(api, [inplace, ok], good) == abi.OK
    # export: JR_E_CAPACITY with the number needed, the descriptors filled either way
    targets = [(g, n) for g in range(G) for n in range(1, R + 1)]
    n = len(targets)
    gs = (C.c_uint32 * n)(*[t[0] for t in targets])
    ns = (C.c_uint32 * n)(*[t[1] for t in targets])
    fn = api._fn("chain_export_many")
    want = api.chain_export_many(targets)
    total = sum(len(b) for _, _, b in want)
    for buf, cap_blocks in ((None, 0), ((abi.Block * total)(), total - 1)):
        desc, need = (abi.PersistedChain * n)(), C.c_size_t(0)
        assert fn(api._h, gs, ns, C.c_size_t(n), desc, buf, C.c_size_t(cap_blocks), C.byref(need)) == abi.E_CAPACITY
        assert need.value == total
        at = 0
        for i, (c, ck, b) in enumerate(want):
            d = desc[i]
            assert (d.group, d.node, d.commit, bool(d.commit_key), d.first_block, d.n_blocks) == (*targets[i], c, ck, at, len(b))
            at += len(b)
    bad_g = (C.c_uint32 * 1)(G)
    assert fn(api._h, bad_g, ns, C.c_size_t(1), desc, None, C.c_size_t(0), C.byref(need)) == abi.E_INVAL


def case_fold_restarts(make, G=40, R=5):
    """Folding engine, non-folding engine and oracle after every launch: followers of half the groups restarted in the
    middle of steady state (from exports and in place), then a leader, which faults on its first append (N2)."""
    apis = trio(make, G, R, seed=R, chain_capacity=512, fsm_units=256)
    for api in apis:
        _bootstrap(api, G, R)
    now = [100]

    def launch(ticks=24):
        for api in apis:
            api.run(now[0], 100, ticks, 1)
        now[0] += 100 * ticks
        same(apis)

    launch()
    launch()
    assert apis[0].fold_count() == G
    half = [(g, n) for g in range(0, G, 2) for n in range(2, R + 1)]
    for api in apis:
        exp = api.chain_export_many(half)
        api.node_restart_many(now[0], [(g, n, bl, c, ck) if g % 4 == 0 else (g, n, None, 0, None)
                                       for (g, n), (c, ck, bl) in zip(half, exp)])
    same(apis)
    for _ in range(3):
        launch()
    assert apis[0].fold_count() > 0
    for api in apis:
        (c, ck, bl), = api.chain_export_many([(1, 1)])
        api.node_restart_many(now[0], [(1, 1, bl, c, ck)])
        api.step(now[0], flags=0, inject=[Command.timeout(1, 1)] + [Command.vote_response(1, 1, 1, v, True) for v in (2, 3)])
        api.step(now[0] + 10, flags=0, inject=[Command.client_request(1, 1, token=99)])
        assert api.query(1, 1).fault == abi.FAULT_APPEND_ID_NOT_GT_HEAD
    now[0] += 100
    same(apis)
    launch()
    launch()


# ---- CPU: the device code -------------------------------------------------------------------------------------------

@pytest.mark.parametrize("R", [3, 5, 7])
def test_export_and_restart_on_device_code(R):
    case_export_and_restart(_emu, R)


@pytest.mark.parametrize("R", [3, 5])
def test_export_and_restart_strict_commit_key_on_device_code(R):
    case_export_and_restart(_emu, R, strict=True, seed=8)


@pytest.mark.parametrize("R", [3, 5, 7])
def test_in_place_equals_export_on_device_code(R):
    case_in_place_equals_export(_emu, R)


def test_commit_without_key_on_device_code():
    case_commit_without_key(_emu)


def test_rejections_on_device_code():
    case_rejections(_emu)


def test_fold_restarts_on_device_code():
    case_fold_restarts(_emu)


def test_export_and_restart_on_oracle_fallback():
    """The oracle has no batched calls: RaftApi loops over its single ones, and persist goes through the same path."""
    api = _oracle(3, 3, seed=6, chain_capacity=32)
    _bootstrap(api, 3, 3)
    api.run(100, 100, 12, 1)
    trees = persist.export_many(api, [(g, 2) for g in range(3)], {})
    persist.restart_many_from_records(api, 2000, trees)
    for g in range(3):
        st = api.query(g, 2)
        assert persist.chain_records(api, g, 2, {}) == trees[(g, 2)]
        assert (st.election_time_ms, st.role, st.head) == (2000, abi.ROLE_FOLLOWER, st.commit)


def test_persisted_chain_size_matches_header(tmp_path):
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "josefine_raft_abi.h"\n'
                   'int main(){printf("%zu %zu %zu %zu\\n",sizeof(jr_persisted_chain),offsetof(jr_persisted_chain,first_block),'
                   'offsetof(jr_persisted_chain,commit_key),(size_t)JR_RESTART_IN_PLACE);return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(abi.PersistedChain), abi.PersistedChain.first_block.offset,
                   abi.PersistedChain.commit_key.offset, abi.RESTART_IN_PLACE]
    assert got[0] == 32


# ---- GPU --------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("R", [3, 5, 7])
def test_export_and_restart_on_gpu(R):
    case_export_and_restart(_gpu, R)
    case_export_and_restart(_gpu, R, strict=True, seed=8)


@pytest.mark.gpu
@pytest.mark.parametrize("R", [3, 5, 7])
def test_in_place_equals_export_on_gpu(R):
    case_in_place_equals_export(_gpu, R)


@pytest.mark.gpu
def test_commit_without_key_and_rejections_on_gpu():
    case_commit_without_key(_gpu)
    case_rejections(_gpu)


@pytest.mark.gpu
def test_fold_restarts_on_gpu():
    case_fold_restarts(_gpu, G=3000)


@pytest.mark.gpu
def test_full_size_bulk_restart_65536x5():
    """65,536 x 5, symmetric-group fold on, auto-truncate 8: node 2 of every group restarted from its export and node 3
    in place, in ONE call, then 128 more ticks -- digests, leader table and sampled states equal the oracle's."""
    G, R = 65536, 5
    cfg = dict(seed=1, chain_capacity=512)
    eng, ora = _gpu(G, R, **cfg), _oracle(G, R, **cfg)
    now = 100
    for api in (eng, ora):
        _bootstrap(api, G, R)
        api.set_auto_truncate(8)
        for k in range(4):
            api.run(now + 6400 * k, 100, 64, 1)
    now += 4 * 6400
    assert eng.fold_count() == G
    assert eng.state_digest() == ora.state_digest()
    exp = eng.chain_export_many([(g, 2) for g in range(G)])
    sample = range(0, G, 4099)
    assert [exp[g] for g in sample] == ora.chain_export_many([(g, 2) for g in sample])
    chains = [(g, 2, bl, c, ck) for g, (c, ck, bl) in enumerate(exp)] + [(g, 3, None, 0, None) for g in range(G)]
    for api in (eng, ora):
        api.node_restart_many(now, chains)
    assert eng.state_digest() == ora.state_digest()
    parity.compare_states(eng, ora, groups=sample, chain_ids=0, where="[restarted]")
    # (restarted followers come back with voted_for None while the others keep the leader's id: no group is symmetric
    # any more, so these ticks run through step_kernel)
    for k in range(2):
        for api in (eng, ora):
            api.run(now + 6400 * k, 100, 64, 1)
    assert eng.state_digest() == ora.state_digest()
    assert eng.leader_table() == ora.leader_table()
    parity.compare_states(eng, ora, groups=sample, chain_ids=0, where="[128 ticks later]")
    reqs = [(g, n, int(eng.query(g, n).chain_floor), 24) for g in sample for n in (2, 3)]
    assert eng.chain_read_many(reqs) == ora.chain_read_many(reqs)
    assert eng.fault_count() == ora.fault_count() == 0
