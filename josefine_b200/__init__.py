"""josefine_b200 -- H100-native batched Chained-Raft engine behind josefine's Raft step API.

Only the hot path of tychedelia/josefine's src/raft (SURVEY.md section 8) lives
here: csrc/ holds the sm_90a kernels and the C ABI (include/josefine_raft_abi.h),
raft.py the host-side mirror of the reference's Command / Apply interface.
"""
from . import abi  # noqa: F401
from .fsm import BatchedDriver, ClientResponse  # noqa: F401
from .raft import (Address, Command, RaftApi, RaftEngine, RaftError, ReplicaHandle,  # noqa: F401
                   StepResult, expand_responses, fsm_tuple, link_cut, load_engine_library, msg_tuple, partition)

__all__ = ["abi", "BatchedDriver", "ClientResponse", "Address", "Command", "RaftApi", "RaftEngine", "RaftError", "ReplicaHandle",
           "StepResult", "expand_responses", "fsm_tuple", "msg_tuple", "load_engine_library", "link_cut", "partition"]
