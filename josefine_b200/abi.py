"""ctypes mirror of include/josefine_raft_abi.h.

The structs here must stay byte-identical to the header; tests/test_abi.py checks
sizes and that the shared library exports every declared symbol.
"""
from __future__ import annotations

import ctypes as C

ABI_VERSION = 2
MAX_REPLICAS = 8
MAX_AE_BLOCKS = 5
MAX_NODE_ID = 65534
CLIENT_QUEUE_CAP = 4
NOTIFY_RUNS = 8           # JR_NOTIFY_RUNS: pending-notification runs per replica (F_CLIENT_RESPONSES)

# jr_status
OK, E_INVAL, E_NOMEM, E_CUDA, E_CAPACITY, E_UNKNOWN_NODE, E_NO_DEVICE = range(7)
STATUS_NAMES = ["JR_OK", "JR_E_INVAL", "JR_E_NOMEM", "JR_E_CUDA", "JR_E_CAPACITY",
                "JR_E_UNKNOWN_NODE", "JR_E_NO_DEVICE"]

# roles (src/raft/mod.rs:403-407)
ROLE_FOLLOWER, ROLE_CANDIDATE, ROLE_LEADER = 0, 1, 2

# Command discriminants (src/raft/mod.rs:160-227)
(CMD_TICK, CMD_PROPOSE, CMD_VOTE_REQUEST, CMD_VOTE_RESPONSE, CMD_APPEND_ENTRIES,
 CMD_APPEND_RESPONSE, CMD_HEARTBEAT, CMD_HEARTBEAT_RESPONSE, CMD_TIMEOUT, CMD_NOOP,
 CMD_CLIENT_REQUEST, CMD_CLIENT_RESPONSE) = range(12)

# Address (src/raft/rpc.rs:5-14)
ADDR_PEERS, ADDR_PEER, ADDR_LOCAL, ADDR_CLIENT = range(4)

# faults
FAULT_NONE = 0
FAULT_AE_STALE_LEADER = 1
FAULT_EXTEND_PARENT_MISSING = 2
FAULT_APPEND_ID_NOT_GT_HEAD = 3
FAULT_COMMIT_BLOCK_MISSING = 4
FAULT_PROGRESS_UNKNOWN_NODE = 5
FAULT_LEADER_TERM_UNIMPLEMENTED = 6
FAULT_CANDIDATE_TICK_ELECTED = 7
FAULT_RANGE_COMMIT_KEY = 8
FAULT_ENGINE_CHAIN_CAPACITY = 64
FAULT_ENGINE_MAILBOX_OVERFLOW = 65
FAULT_ENGINE_FSM_OVERFLOW = 66
FAULT_ENGINE_QUEUE_OVERFLOW = 67

# engine flags
F_SLED_COMMIT_KEY_STRICT = 1 << 0
F_CAPTURE_MESSAGES = 1 << 1
F_CAPTURE_FSM = 1 << 2
F_STREAM_DIGEST = 1 << 3
F_NO_SYMMETRIC_FOLD = 1 << 4
F_CLIENT_RESPONSES = 1 << 5

# step flags
STEP_DELIVER = 1 << 0
STEP_TICK = 1 << 1
STEP_SYNTH_PROPOSALS = 1 << 2
STEP_TRUSTED_PROPOSALS = 1 << 3
STEP_REPORT_FAULTS = 1 << 4

FSM_APPLY, FSM_NOTIFY = 0, 1


class Config(C.Structure):
    _fields_ = [
        ("abi_version", C.c_uint32), ("n_groups", C.c_uint32), ("n_replicas", C.c_uint32),
        ("device", C.c_int32), ("seed", C.c_uint64), ("group_offset", C.c_uint64),
        ("election_min_ms", C.c_uint32), ("election_max_ms", C.c_uint32),
        ("heartbeat_ms", C.c_uint32), ("chain_capacity", C.c_uint32),
        ("mailbox_units", C.c_uint32), ("fsm_units", C.c_uint32),
        ("flags", C.c_uint32), ("resident_mask", C.c_uint32),
        ("fsm_host_records", C.c_uint32), ("fsm_raw_units", C.c_uint32),
    ]


class Block(C.Structure):
    _fields_ = [("id", C.c_uint64), ("next", C.c_uint64), ("data", C.c_uint64)]


class Msg(C.Structure):
    _fields_ = [
        ("group", C.c_uint32),
        ("from_kind", C.c_uint8), ("to_kind", C.c_uint8), ("kind", C.c_uint8), ("flag", C.c_uint8),
        ("from_id", C.c_uint32), ("to_id", C.c_uint32), ("node_id", C.c_uint32),
        ("n_blocks", C.c_uint8), ("client_kind", C.c_uint8), ("reserved", C.c_uint16),
        ("client_id", C.c_uint32), ("reserved2", C.c_uint32),
        ("term", C.c_uint64), ("last_term", C.c_uint64), ("block", C.c_uint64), ("token", C.c_uint64),
        ("blocks", Block * MAX_AE_BLOCKS),
    ]


class FsmInstr(C.Structure):
    _fields_ = [
        ("group", C.c_uint32), ("node", C.c_uint32),
        ("kind", C.c_uint8), ("client_kind", C.c_uint8), ("reserved", C.c_uint16),
        ("client_id", C.c_uint32),
        ("block", Block),
    ]


class Proposal(C.Structure):
    _fields_ = [("token", C.c_uint64), ("node", C.c_uint32), ("reserved", C.c_uint32)]


class TokenRun(C.Structure):
    _fields_ = [("base", C.c_uint64), ("stride", C.c_uint64)]


class StepArgs(C.Structure):
    _fields_ = [
        ("now_ms", C.c_uint64), ("flags", C.c_uint32), ("n_synth", C.c_uint32),
        ("inject", C.POINTER(Msg)), ("n_inject", C.c_size_t),
        ("proposals", C.POINTER(Proposal)),
        ("out_msgs", C.POINTER(Msg)), ("cap_msgs", C.c_size_t), ("n_msgs", C.c_size_t),
        ("out_fsm", C.POINTER(FsmInstr)), ("cap_fsm", C.c_size_t), ("n_fsm", C.c_size_t),
        ("n_faulted", C.c_uint64),
    ]


class ReplicaState(C.Structure):
    _fields_ = [
        ("current_term", C.c_uint64), ("voted_for", C.c_uint32), ("leader_id", C.c_uint32),
        ("election_time_ms", C.c_uint64), ("election_timeout_ms", C.c_uint32), ("rng_draws", C.c_uint32),
        ("head", C.c_uint64), ("commit", C.c_uint64), ("id_gen", C.c_uint64), ("max_key", C.c_uint64),
        ("heartbeat_time_ms", C.c_uint64), ("votes_seen", C.c_uint32), ("votes_granted", C.c_uint32),
        ("progress_head", C.c_uint64 * MAX_REPLICAS), ("progress_replicate", C.c_uint32),
        ("role", C.c_uint8), ("fault", C.c_uint8), ("alive", C.c_uint8), ("n_queued", C.c_uint8),
        ("chain_floor", C.c_uint64),
    ]

    def as_dict(self) -> dict:
        d = {}
        for name, _ in self._fields_:
            v = getattr(self, name)
            d[name] = list(v) if hasattr(v, "__len__") else v
        return d


FSMR_APPLY, FSMR_NOTIFY, FSMR_PATTERN, FSMR_RESPONSE = 0, 1, 2, 3


class FsmRecord(C.Structure):
    """jr_fsm_record: one run of a replica's Instruction stream (layout normative in the header)."""
    _fields_ = [("group", C.c_uint32), ("hdr", C.c_uint32), ("id0", C.c_uint32), ("addr", C.c_uint32),
                ("tok0", C.c_uint64), ("stride", C.c_uint64)]

    @property
    def kind(self) -> int:
        return self.hdr & 3

    @property
    def node(self) -> int:
        return ((self.hdr >> 2) & 7) + 1

    @property
    def count(self) -> int:
        return self.hdr >> 8


class FsmBatch(C.Structure):
    _fields_ = [("n_records", C.c_uint64), ("n_dropped", C.c_uint64), ("n_instructions", C.c_uint64),
                ("node_offset", C.c_uint32 * (MAX_REPLICAS + 1)), ("reserved", C.c_uint32)]


class LeaderEntry(C.Structure):
    _fields_ = [("term", C.c_uint64), ("leader_id", C.c_uint32), ("commit", C.c_uint32)]


RESTART_IN_PLACE = 0xFFFFFFFF


class PersistedChain(C.Structure):
    """jr_persisted_chain: one replica's sled tree -- blocks[first_block : first_block + n_blocks] and the commit key."""
    _fields_ = [("group", C.c_uint32), ("node", C.c_uint32), ("commit", C.c_uint64), ("first_block", C.c_uint64),
                ("n_blocks", C.c_uint32), ("commit_key", C.c_uint32)]


# jr_verify_groups finding kinds (normative rules in the header)
VERIFY_BELOW_FLOOR, VERIFY_COMMIT_ABSENT, VERIFY_CHAIN_BROKEN, VERIFY_DIVERGED, VERIFY_LEADER_CONFLICT = 1, 2, 3, 4, 5
VERIFY_KIND_NAMES = {1: "BELOW_FLOOR", 2: "COMMIT_ABSENT", 3: "CHAIN_BROKEN", 4: "DIVERGED", 5: "LEADER_CONFLICT"}


class VerifyReport(C.Structure):
    """jr_verify_report: what one jr_verify_groups call checked, and its findings per kind."""
    _fields_ = [("groups_checked", C.c_uint64), ("replicas_checked", C.c_uint64), ("replicas_skipped", C.c_uint64),
                ("below_floor", C.c_uint64), ("commit_absent", C.c_uint64), ("chain_broken", C.c_uint64),
                ("diverged", C.c_uint64), ("leader_conflicts", C.c_uint64)]

    def as_tuple(self) -> tuple:
        return tuple(getattr(self, k) for k, _ in self._fields_)


class VerifyFinding(C.Structure):
    """jr_verify_finding: one replica that is not OK, or one (group, term) with two or more leaders (node 0)."""
    _fields_ = [("group", C.c_uint32), ("kind", C.c_uint8), ("node", C.c_uint8), ("ref_node", C.c_uint8),
                ("node_mask", C.c_uint8), ("id", C.c_uint64), ("term", C.c_uint64), ("reserved", C.c_uint64)]

    def as_tuple(self) -> tuple:
        return (self.group, self.kind, self.node, self.ref_node, self.node_mask, self.id, self.term)


# sizes the header implies (checked in tests/test_abi.py against offsetof-free arithmetic)
EXPECTED_SIZES = {
    "Config": 72, "Block": 24, "Msg": 64 + 24 * MAX_AE_BLOCKS, "FsmInstr": 16 + 24,
    "Proposal": 16, "TokenRun": 16, "LeaderEntry": 16, "FsmRecord": 32, "FsmBatch": 24 + 4 * (MAX_REPLICAS + 1) + 4,
    "ReplicaState": 160, "PersistedChain": 32, "VerifyReport": 64, "VerifyFinding": 32,
}

# every symbol include/josefine_raft_abi.h declares
ENGINE_SYMBOLS = [
    "jr_engine_create", "jr_engine_destroy", "jr_engine_reset", "jr_engine_set_stream", "jr_engine_sync",
    "jr_last_error", "jr_config_default", "jr_step", "jr_run", "jr_run_proposals", "jr_run_tokens", "jr_run_token_runs", "jr_drain_fsm", "jr_query",
    "jr_chain_read", "jr_state_digest", "jr_stream_digest", "jr_fault_count", "jr_fold_count", "jr_compact",
    "jr_set_alive", "jr_kill_leaders", "jr_leader_table_device", "jr_leader_table", "jr_leader_table_async", "jr_leader_table_wait",
    "jr_election_timeout", "jr_fsm_records_async", "jr_fsm_records_wait", "jr_fsm_responses", "jr_fsm_expand", "jr_fsm_fold", "jr_fsm_fold_mt", "jr_query_many",
    "jr_chain_read_many", "jr_truncate", "jr_set_auto_truncate", "jr_host_alloc", "jr_host_free", "jr_node_restart", "jr_chain_export_many", "jr_node_restart_many", "jr_verify_groups", "jr_engine_save_size", "jr_engine_save", "jr_engine_restore",
]


def default_config(n_groups: int, n_replicas: int, **kw) -> Config:
    """jr_config_default in Python (same numbers; kept in sync by tests/test_abi.py)."""
    cfg = Config()
    cfg.abi_version = ABI_VERSION
    cfg.n_groups = n_groups
    cfg.n_replicas = n_replicas
    cfg.device = 0
    cfg.seed = 0
    cfg.group_offset = 0
    cfg.election_min_ms = 500      # src/raft/mod.rs:318
    cfg.election_max_ms = 1000     # src/raft/mod.rs:319
    cfg.heartbeat_ms = 100         # src/raft/config.rs:104
    cfg.chain_capacity = 4096
    cfg.mailbox_units = 64
    cfg.fsm_units = 64
    cfg.flags = 0
    cfg.fsm_host_records = 0
    for k, v in kw.items():
        if not hasattr(cfg, k):
            raise AttributeError(k)
        setattr(cfg, k, v)
    return cfg
