"""GPU suite: the CUDA engine, called through the C ABI (libjosefine_b200.so),
against the C++ restatement oracle -- bit for bit.  Needs an H100."""
import pytest

from josefine_b200 import abi, RaftEngine
from oracle.restated import RestatedCluster
from tests import kat_cases, parity

pytestmark = pytest.mark.gpu


def make_oracle(g, r, **kw):
    return RestatedCluster.create(g, r, n_threads=16 if g >= 1024 else 1, **kw)


def make_gpu(g, r, **kw):
    return RaftEngine.create(g, r, **kw)


@pytest.mark.parametrize("case", kat_cases.ALL_KATS, ids=lambda f: f.__name__)
def test_reference_kat_on_gpu(case):
    case(make_gpu)


@pytest.mark.parametrize("R", [1, 2, 3, 4, 5, 6, 7, 8])
def test_cold_start(R):
    p = parity.Pair(make_oracle, make_gpu, 40, R, seed=R, check_states_every=5)
    parity.scenario_cold_start(p, steps=45)


@pytest.mark.parametrize("R", [3, 5, 7])
def test_steady_state(R):
    p = parity.Pair(make_oracle, make_gpu, 33, R, seed=1, check_states_every=4)
    parity.scenario_steady(p, steps=24)


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("R", [3, 5, 7])
def test_random_inject(R, seed):
    p = parity.Pair(make_oracle, make_gpu, 5, R, seed=seed, chain_capacity=64, check_states_every=10)
    parity.scenario_random_inject(p, seed=seed * 7 + R, steps=50)


@pytest.mark.parametrize("R", [3, 5])
def test_random_inject_strict_commit_key(R):
    p = parity.Pair(make_oracle, make_gpu, 5, R, seed=5, chain_capacity=64, check_states_every=10,
                    flags=parity.FULL | abi.F_SLED_COMMIT_KEY_STRICT)
    parity.scenario_random_inject(p, seed=99 + R, steps=50)


def test_run_equals_steps():
    a = make_gpu(100, 3, seed=3, flags=parity.FULL)
    b = make_gpu(100, 3, seed=3, flags=parity.FULL)
    a.run(100, 100, 30, 1)
    for k in range(30):
        b.step(100 + 100 * k, n_synth=1)
    parity.compare_states(a, b, groups=range(0, 100, 7), chain_ids=40)
    parity.compare_digests(a, b)


def _digest_parity(G, R, steps, seed, bootstrap, n_synth=1, sample=16, **kw):
    """Full-size check through size-independent digests (a checksum of per-replica
    checksums of every Message / Instruction / state word) plus exact state on a sample."""
    flags = abi.F_STREAM_DIGEST
    a = make_oracle(G, R, seed=seed, flags=flags, **kw)
    b = make_gpu(G, R, seed=seed, flags=flags, **kw)
    if bootstrap:
        from josefine_b200 import Command
        inj = []
        q = R // 2 + 1
        for g in range(G):
            inj.append(Command.timeout(g, 1))
            for v in range(2, q + 1):
                inj.append(Command.vote_response(g, 1, 1, v, True))
        a.step(0, flags=0, inject=inj)
        b.step(0, flags=0, inject=inj)
    a.run(100, 100, steps, n_synth)
    b.run(100, 100, steps, n_synth)
    parity.compare_digests(a, b, f"[{G}x{R} after {steps} steps]")
    step = max(G // sample, 1)
    parity.compare_states(a, b, groups=range(0, G, step), chain_ids=min(steps + 4, 64))
    assert a.leader_table() == b.leader_table()
    return a, b


def test_config2_1024x3_vote_append():
    """BASELINE config #2: 1,024 groups x 3 replicas, cold start, elections, then proposals."""
    a, b = _digest_parity(1024, 3, 256, seed=0, bootstrap=False, chain_capacity=512)
    leaders = [l for (_, l, _) in b.leader_table()]
    assert sum(1 for l in leaders if l) > 900  # nearly every group elected someone


def test_config3_65536x5_steady_append():
    """BASELINE config #3 at full size: 65,536 x 5, pre-elected leaders, steady AppendEntries."""
    a, b = _digest_parity(65536, 5, 48, seed=1, bootstrap=True, chain_capacity=128)
    assert all(l == 1 for (_, l, _) in b.leader_table()[:100])
    assert b.fault_count() == 0


def test_config5_7_replicas_churn_and_compact():
    """BASELINE config #5 shape (reduced G): 7 replicas, leader loss, compact()."""
    G, R = 4096, 7
    flags = abi.F_STREAM_DIGEST
    a = make_oracle(G, R, seed=2, flags=flags, chain_capacity=256)
    b = make_gpu(G, R, seed=2, flags=flags, chain_capacity=256)
    from josefine_b200 import Command
    inj = []
    for g in range(G):
        inj.append(Command.timeout(g, 1))
        for v in (2, 3, 4):
            inj.append(Command.vote_response(g, 1, 1, v, True))
    for x in (a, b):
        x.step(0, flags=0, inject=inj)
    now = 100
    for rnd in range(3):
        for x in (a, b):
            x.run(now, 100, 40, 1)
        now += 4000
        ka, kb = a.kill_leaders(rnd, 100), b.kill_leaders(rnd, 100)
        assert ka == kb
        for x in (a, b):
            x.compact()
        parity.compare_digests(a, b, f"[churn round {rnd}]")
    parity.compare_states(a, b, groups=range(0, G, 257), chain_ids=64)
    # SURVEY N1: followers keep voted_for = dead leader, so killed groups stay leaderless
    dead = sum(1 for (_, l, _) in b.leader_table() if l == 0)
    assert dead > 0


def test_no_cpu_fallback_symbols():
    """The product library must be the CUDA one: it reports a device-side digest that
    only the kernels can produce, and the oracle library is not loaded by the package."""
    import josefine_b200.raft as r
    assert r.ENGINE_LIB_PATH.endswith("libjosefine_b200.so")
    e = make_gpu(8, 3)
    assert e.state_digest() != 0


def test_config4_per_gpu_shard_131072x5():
    """BASELINE config #4's per-GPU share (1,048,576 / 8 = 131,072 groups x 5), as the shard of
    rank 3: group_offset keeps the D2 timeouts keyed by GLOBAL group id."""
    G = 131072
    a, b = _digest_parity(G, 5, 24, seed=1, bootstrap=True, chain_capacity=64, group_offset=3 * G)
    assert b.fault_count() == 0


def test_config5_full_size_65536x7_churn_compact():
    """BASELINE config #5 at full size: 65,536 x 7, leaders silenced in 10% of the groups, compact()."""
    G, R = 65536, 7
    flags = abi.F_STREAM_DIGEST
    a = make_oracle(G, R, seed=2, flags=flags, chain_capacity=96)
    b = make_gpu(G, R, seed=2, flags=flags, chain_capacity=96)
    from josefine_b200 import Command
    inj = []
    for g in range(G):
        inj.append(Command.timeout(g, 1))
        for v in (2, 3, 4):
            inj.append(Command.vote_response(g, 1, 1, v, True))
    for x in (a, b):
        x.step(0, flags=0, inject=inj)
    now = 100
    for rnd in range(2):
        for x in (a, b):
            x.run(now, 100, 20, 1)
        now += 2000
        assert a.kill_leaders(rnd, 100) == b.kill_leaders(rnd, 100)
        for x in (a, b):
            x.compact()
    parity.compare_digests(a, b, "[65536x7 churn]")
    parity.compare_states(a, b, groups=range(0, G, 4099), chain_ids=48)
    table = b.leader_table()
    assert table == a.leader_table()
    assert 0.05 < sum(1 for (_, l, _) in table if l == 0) / G < 0.30


@pytest.mark.parametrize("variant", ["plain", "sorted"])
def test_kernel_variants_scattered_leaders(monkeypatch, variant):
    """Leaders spread over all replica indices (what real elections produce): the plain and the
    role-sorted kernel variant both match the oracle at 8,192 x 5."""
    monkeypatch.setenv("JR_STEP_VARIANT", variant)
    from josefine_b200 import Command
    G, R = 8192, 5
    flags = abi.F_STREAM_DIGEST
    a = make_oracle(G, R, seed=6, flags=flags, chain_capacity=128)
    b = make_gpu(G, R, seed=6, flags=flags, chain_capacity=128)
    inj = []
    for g in range(G):
        n = g % R + 1
        inj.append(Command.timeout(g, n))
        for v in [v for v in range(1, R + 1) if v != n][:2]:
            inj.append(Command.vote_response(g, n, 1, v, True))
    for x in (a, b):
        x.step(0, flags=0, inject=inj)
        x.run(100, 100, 40, 1)
        x.run(4100, 100, 9, 2)
    parity.compare_digests(a, b, f"[scattered leaders, {variant}]")
    parity.compare_states(a, b, groups=range(0, G, 331), chain_ids=64)
    assert sorted({l for (_, l, _) in b.leader_table()}) == [1, 2, 3, 4, 5]


def test_config3_soak_256_ticks():
    """Config #3 at full size for 256 ticks in four fused launches (the bench's launch shape)."""
    G, R = 65536, 5
    flags = abi.F_STREAM_DIGEST
    a = make_oracle(G, R, seed=1, flags=flags, chain_capacity=320)
    b = make_gpu(G, R, seed=1, flags=flags, chain_capacity=320)
    from josefine_b200 import Command
    inj = []
    for g in range(G):
        inj.append(Command.timeout(g, 1))
        for v in (2, 3):
            inj.append(Command.vote_response(g, 1, 1, v, True))
    for x in (a, b):
        x.step(0, flags=0, inject=inj)
    now = 100
    for chunk in range(4):
        for x in (a, b):
            x.run(now, 100, 64, 1)
        now += 6400
    parity.compare_digests(a, b, "[65536x5, 256 ticks]")
    parity.compare_states(a, b, groups=range(0, G, 5003), chain_ids=64)
    assert b.fault_count() == 0 and min(c for (_, _, c) in b.leader_table()) > 240


def test_long_run_1024_ticks_with_two_proposals_per_tick():
    G, R = 2048, 5
    flags = abi.F_STREAM_DIGEST
    a = make_oracle(G, R, seed=12, flags=flags, chain_capacity=2200)
    b = make_gpu(G, R, seed=12, flags=flags, chain_capacity=2200)
    from josefine_b200 import Command
    inj = []
    for g in range(G):
        inj.append(Command.timeout(g, 2))
        for v in (1, 3):
            inj.append(Command.vote_response(g, 2, 1, v, True))
    for x in (a, b):
        x.step(0, flags=0, inject=inj)
        x.run(100, 100, 1024, 2)
    parity.compare_digests(a, b, "[2048x5, 1024 ticks, 2 proposals/tick]")
    assert b.fault_count() == 0 and max(c for (_, _, c) in b.leader_table()) > 2000


def test_three_single_node_engines_over_the_wire_match_resident_cluster():
    """INTEGRATION.md section 1 arrangement: one hosted node per engine (resident_mask), peers reached through
    josefine's TCP framing (josefine_b200/wire.py; tcp.rs:39-51,143-156) -- must equal the co-resident group."""
    from tests.wire_cluster import run_networked_vs_resident
    frames, nbytes = run_networked_vs_resident(make_gpu)
    assert frames > 100 and nbytes > frames * 60


def test_leader_routed_tokens():
    parity.scenario_leader_routed_tokens(make_gpu, make_oracle)


def test_leader_routed_tokens_many_groups():
    parity.scenario_leader_routed_tokens(make_gpu, make_oracle, G=3000, R=3, seed=2)


@pytest.mark.parametrize("parts", [2, 3, 8])
def test_split_launches_are_bit_identical(monkeypatch, parts):
    """A launch cut into ticket-ordered tasks (DESIGN.md section 3, "Split launches") -- here forced, at a size where
    the tasks of one block really run on different SMs at different times -- equals the unsplit launch and the oracle."""
    G, R = 8192, 3
    monkeypatch.setenv("JR_PARTS", str(parts))
    split = make_gpu(G, R, seed=9, flags=abi.F_STREAM_DIGEST)
    monkeypatch.setenv("JR_PARTS", "1")
    whole = make_gpu(G, R, seed=9, flags=abi.F_STREAM_DIGEST)
    o = make_oracle(G, R, seed=9, flags=abi.F_STREAM_DIGEST)
    for eng in (split, whole, o):
        eng.run(100, 100, 23, 0)
        eng.run(2400, 100, 37, 2)
        eng.leader_table()
        eng.run_tokens(6100, 100, [[(k << 20) | (g + 1) for g in range(G)] for k in range(9)])
    assert split.state_digest() == whole.state_digest() == o.state_digest()
    assert split.stream_digest() == whole.stream_digest() == o.stream_digest()
    assert split.leader_table() == whole.leader_table() == o.leader_table()
    assert split.fault_count() == o.fault_count()
