//! josefine_gpu_shim.rs -- Rust side of the drop-in boundary (SURVEY.md section 8f, row 1).
//!
//! **UNTESTED SOURCE.**  The build environment of this repository has no `cargo` / `rustc`, so
//! this file has never been compiled.  It shows, concretely, what a josefine maintainer would
//! add to `src/raft/` to drive `libjosefine_b200.so` through `include/josefine_raft_abi.h`:
//! `#[repr(C)]` mirrors of the POD structs, the `extern "C"` block, `Command <-> jr_msg`
//! conversion, and an `event_loop` whose five `raft.apply(..)` sites (src/raft/server.rs:125,
//! 133,135,143,159) each become ONE `jr_step`: the tick site steps with DELIVER|TICK, the inbound-RPC
//! and client sites step with flags = 0 and the one command injected, so a command is applied the
//! moment it arrives, exactly as `raft.apply(cmd)` does in the reference.  The Python binding in
//! `josefine_b200/raft.py` is the one the tests exercise; field order and sizes here follow the
//! same header and are checked on the C side by `tests/test_abi.py`.
//!
//! Mapping (reference item -> here):
//!   RaftHandle::new                   mod.rs:428-435     -> GpuRaft::new (jr_engine_create, resident_mask = this node)
//!   Apply::apply(Command::Tick)       server.rs:125      -> GpuRaft::tick (jr_step DELIVER|TICK)
//!   apply(msg.command) from tcp_rx    server.rs:127-137  -> GpuRaft::on_peer_message (jr_step, flags 0, inject = [msg]: applied at once)
//!   apply(ClientRequest)              server.rs:156-160  -> GpuRaft::propose        (jr_step, flags 0, inject = [ClientRequest])
//!   rpc_tx.send(Message)              mod.rs:390-400     -> StepOutput::messages
//!   fsm_tx.send(Instruction)          leader.rs:94,184   -> StepOutput::instructions
//!   panic!/Err in the state machine   (see JR_FAULT_*)   -> StepOutput::faulted (jr_step_args.n_faulted, JR_STEP_REPORT_FAULTS)
//!                                                           -> event_loop returns Err; no jr_query per step

#![allow(dead_code)]

use std::collections::HashMap;
use std::os::raw::{c_char, c_int, c_void};

use crate::raft::chain::{Block, BlockId};
use crate::raft::fsm::Instruction;
use crate::raft::rpc::{Address, Message, Proposal};
use crate::raft::{ClientRequest, ClientRequestId, Command, NodeId};

// ---- POD mirrors of include/josefine_raft_abi.h ------------------------------------------------

pub const JR_ABI_VERSION: u32 = 2;
pub const JR_MAX_AE_BLOCKS: usize = 5;
pub const JR_F_CAPTURE_MESSAGES: u32 = 1 << 1;
pub const JR_F_CAPTURE_FSM: u32 = 1 << 2;
pub const JR_STEP_DELIVER: u32 = 1 << 0;
pub const JR_STEP_TICK: u32 = 1 << 1;
pub const JR_STEP_REPORT_FAULTS: u32 = 1 << 4;

#[repr(C)]
#[derive(Clone, Copy, Default)]
pub struct JrConfig {
    pub abi_version: u32,
    pub n_groups: u32,
    pub n_replicas: u32,
    pub device: i32,
    pub seed: u64,
    pub group_offset: u64,
    pub election_min_ms: u32,
    pub election_max_ms: u32,
    pub heartbeat_ms: u32,
    pub chain_capacity: u32,
    pub mailbox_units: u32,
    pub fsm_units: u32,
    pub flags: u32,
    pub resident_mask: u32,
    pub fsm_host_records: u32,
    pub fsm_raw_units: u32,
}

#[repr(C)]
#[derive(Clone, Copy, Default)]
pub struct JrBlock {
    pub id: u64,
    pub next: u64,
    pub data: u64, // payload token (deviation D5)
}

#[repr(C)]
#[derive(Clone, Copy, Default)]
pub struct JrMsg {
    pub group: u32,
    pub from_kind: u8,
    pub to_kind: u8,
    pub kind: u8,
    pub flag: u8,
    pub from_id: u32,
    pub to_id: u32,
    pub node_id: u32,
    pub n_blocks: u8,
    pub client_kind: u8,
    pub reserved: u16,
    pub client_id: u32,
    pub reserved2: u32,
    pub term: u64,
    pub last_term: u64,
    pub block: u64,
    pub token: u64,
    pub blocks: [JrBlock; JR_MAX_AE_BLOCKS],
}

#[repr(C)]
#[derive(Clone, Copy, Default)]
pub struct JrFsmInstr {
    pub group: u32,
    pub node: u32,
    pub kind: u8, // 0 Apply, 1 Notify
    pub client_kind: u8,
    pub reserved: u16,
    pub client_id: u32,
    pub block: JrBlock,
}

#[repr(C)]
#[derive(Clone, Copy, Default)]
pub struct JrProposal {
    pub token: u64,
    pub node: u32,
    pub reserved: u32,
}

#[repr(C)]
pub struct JrStepArgs {
    pub now_ms: u64,
    pub flags: u32,
    pub n_synth: u32,
    pub inject: *const JrMsg,
    pub n_inject: usize,
    pub proposals: *const JrProposal,
    pub out_msgs: *mut JrMsg,
    pub cap_msgs: usize,
    pub n_msgs: usize,
    pub out_fsm: *mut JrFsmInstr,
    pub cap_fsm: usize,
    pub n_fsm: usize,
    pub n_faulted: u64, // out, with JR_STEP_REPORT_FAULTS
}

#[repr(C)]
#[derive(Clone, Copy)]
pub struct JrReplicaState {
    pub current_term: u64,
    pub voted_for: u32,
    pub leader_id: u32,
    pub election_time_ms: u64,
    pub election_timeout_ms: u32,
    pub rng_draws: u32,
    pub head: u64,
    pub commit: u64,
    pub id_gen: u64,
    pub max_key: u64,
    pub heartbeat_time_ms: u64,
    pub votes_seen: u32,
    pub votes_granted: u32,
    pub progress_head: [u64; 8],
    pub progress_replicate: u32,
    pub role: u8,
    pub fault: u8,
    pub alive: u8,
    pub n_queued: u8,
    pub chain_floor: u64, // deviation D7
}

#[link(name = "josefine_b200")]
extern "C" {
    fn jr_config_default(cfg: *mut JrConfig, n_groups: u32, n_replicas: u32);
    fn jr_engine_create(cfg: *const JrConfig, out: *mut *mut c_void) -> c_int;
    fn jr_engine_destroy(e: *mut c_void);
    fn jr_step(e: *mut c_void, args: *mut JrStepArgs) -> c_int;
    /// n_steps fused ticks; tokens[k * n_groups + g] (0 = none) goes to the leader the last jr_leader_table* call announced.
    #[allow(dead_code)]
    fn jr_run_tokens(e: *mut c_void, now0_ms: u64, dt_ms: u32, n_steps: u32, tokens: *const u64) -> c_int;
    fn jr_query(e: *mut c_void, group: u32, node: u32, out: *mut JrReplicaState) -> c_int;
    fn jr_last_error() -> *const c_char;
    // The batched calls a broker hosting many groups per process would use instead (INTEGRATION.md section 2a;
    // examples/batched_quantum.c is that loop in C).  Declared for completeness: this shim keeps josefine's
    // one-node-per-process shape and does not call them.
    #[allow(dead_code)]
    fn jr_host_alloc(bytes: usize, out: *mut *mut c_void) -> c_int;
    #[allow(dead_code)]
    fn jr_host_free(p: *mut c_void);
    #[allow(dead_code)]
    fn jr_set_auto_truncate(e: *mut c_void, enabled: c_int, margin: u32) -> c_int;
    #[allow(dead_code)]
    fn jr_run_token_runs(e: *mut c_void, now0_ms: u64, dt_ms: u32, n_steps: u32, runs: *const [u64; 2]) -> c_int;
    #[allow(dead_code)]
    fn jr_fsm_records_async(e: *mut c_void) -> c_int;
    #[allow(dead_code)]
    fn jr_fsm_records_wait(e: *mut c_void, records: *mut *const c_void, batch: *mut c_void) -> c_int;
    #[allow(dead_code)]
    fn jr_fsm_responses(e: *mut c_void, responses: *mut *const JrFsmRecord, batch: *mut c_void) -> c_int;
    #[allow(dead_code)]
    fn jr_chain_export_many(e: *mut c_void, groups: *const u32, nodes: *const u32, n: usize, out: *mut JrPersistedChain,
                            blocks: *mut JrBlock, cap_blocks: usize, n_blocks: *mut usize) -> c_int;
    #[allow(dead_code)]
    fn jr_node_restart_many(e: *mut c_void, now_ms: u64, chains: *const JrPersistedChain, n: usize, blocks: *const JrBlock,
                            n_blocks: usize) -> c_int;
    #[allow(dead_code)]
    fn jr_group_export(e: *mut c_void, groups: *const u32, n: usize, image: *mut u8, cap: usize, bytes: *mut usize) -> c_int;
    #[allow(dead_code)]
    fn jr_group_import(e: *mut c_void, slots: *const u32, n: usize, image: *const u8, bytes: usize) -> c_int;
    #[allow(dead_code)]
    fn jr_verify_groups(e: *mut c_void, groups: *const u32, n_groups: usize, report: *mut JrVerifyReport,
                        findings: *mut JrVerifyFinding, cap: usize, n_findings: *mut usize) -> c_int;
    // peer-link cuts (JR_F_PEER_LINKS, deviation D8): bit 8*(r-1) + (s-1) of a group's matrix = mail s -> r is dropped
    #[allow(dead_code)]
    fn jr_set_links(e: *mut c_void, groups: *const u32, cuts: *const u64, n: usize) -> c_int;
    #[allow(dead_code)]
    fn jr_get_links(e: *mut c_void, groups: *const u32, n: usize, out: *mut u64) -> c_int;
    #[allow(dead_code)]
    fn jr_isolate_leaders(e: *mut c_void, salt: u64, permille: u32, n_isolated: *mut u64) -> c_int;
    // link queues (JR_F_LINK_QUEUES): depths[64*i + 8*(r-1) + (s-1)] = Messages queued on link s -> r of groups[i]
    #[allow(dead_code)]
    fn jr_get_link_queues(e: *mut c_void, groups: *const u32, n: usize, depths: *mut u8) -> c_int;
}

/// jr_verify_report: what one jr_verify_groups call checked, and its findings per kind.
#[repr(C)]
#[derive(Clone, Copy, Default, Debug)]
pub struct JrVerifyReport {
    pub groups_checked: u64,
    pub replicas_checked: u64,
    pub replicas_skipped: u64, // silenced or faulted
    pub below_floor: u64,
    pub commit_absent: u64,
    pub chain_broken: u64,
    pub diverged: u64,
    pub leader_conflicts: u64,
}

/// jr_verify_finding (32 B): kind 1 BELOW_FLOOR, 2 COMMIT_ABSENT, 3 CHAIN_BROKEN, 4 DIVERGED, 5 LEADER_CONFLICT (node 0).
#[repr(C)]
#[derive(Clone, Copy, Default, Debug)]
pub struct JrVerifyFinding {
    pub group: u32,
    pub kind: u8,
    pub node: u8,
    pub ref_node: u8,
    pub node_mask: u8,
    pub id: u64,
    pub term: u64,
    pub reserved: u64,
}

/// Sketch: right after `restart_hosted_groups`, check that the reopened replicas hold the committed chain their groups
/// agree on -- a stale, misplaced or corrupt tree shows up as a finding before the broker serves from it.  `groups` are
/// the restarted groups (empty: every group).  Two calls when something is found: the first one sizes the buffer.
#[allow(dead_code)]
unsafe fn verify_restarted_groups(engine: *mut c_void, groups: &[u32]) -> Result<(JrVerifyReport, Vec<JrVerifyFinding>), c_int> {
    let (ptr, n) = if groups.is_empty() { (std::ptr::null(), 0) } else { (groups.as_ptr(), groups.len()) };
    let mut report = JrVerifyReport::default();
    let mut need = 0usize;
    match jr_verify_groups(engine, ptr, n, &mut report, std::ptr::null_mut(), 0, &mut need) {
        0 => return Ok((report, Vec::new())),
        4 => {} // JR_E_CAPACITY: `need` findings
        st => return Err(st),
    }
    let mut findings = vec![JrVerifyFinding::default(); need];
    let st = jr_verify_groups(engine, ptr, n, &mut report, findings.as_mut_ptr(), findings.len(), &mut need);
    if st != 0 {
        return Err(st);
    }
    findings.truncate(need);
    Ok((report, findings))
}

/// One replica's persisted sled tree (chain.rs:99-104): blocks[first_block .. first_block + n_blocks] + the commit key.
#[repr(C)]
#[derive(Clone, Copy, Default)]
pub struct JrPersistedChain {
    pub group: u32,
    pub node: u32,
    pub commit: u64,
    pub first_block: u64,
    pub n_blocks: u32, // JR_RESTART_IN_PLACE: reopen the replica's own table
    pub commit_key: u32,
}
#[allow(dead_code)]
const JR_RESTART_IN_PLACE: u32 = 0xFFFF_FFFF;

/// Sketch: what `Server::run` of a broker hosting node `id` of `n_groups` groups would do at start-up instead of one
/// `RaftHandle::new` per group -- reopen every hosted group from the trees it kept, in ONE call.  `trees[g]` is
/// (commit, commit key present, blocks) as read back from the host's store (`jr_chain_export_many` wrote them).
#[allow(dead_code)]
unsafe fn restart_hosted_groups(engine: *mut c_void, id: u32, now_ms: u64, trees: &[(u64, bool, Vec<JrBlock>)]) -> c_int {
    let mut chains = Vec::with_capacity(trees.len());
    let mut blocks = Vec::new();
    for (g, (commit, key, bl)) in trees.iter().enumerate() {
        chains.push(JrPersistedChain {
            group: g as u32,
            node: id,
            commit: *commit,
            first_block: blocks.len() as u64,
            n_blocks: bl.len() as u32,
            commit_key: *key as u32,
        });
        blocks.extend_from_slice(bl);
    }
    jr_node_restart_many(engine, now_ms, chains.as_ptr(), chains.len(), blocks.as_ptr(), blocks.len())
}

/// jr_fsm_record (32 B); with JR_FSMR_RESPONSE (kind 3) element i answers request token tok0 + i*stride.
#[repr(C)]
#[derive(Clone, Copy, Default)]
pub struct JrFsmRecord {
    pub group: u32,
    pub hdr: u32, // bits 0-1 kind, 2-4 node id - 1, 8-31 count
    pub id0: u32,
    pub addr: u32, // client_kind << 16 | client_id
    pub tok0: u64,
    pub stride: u64,
}
#[allow(dead_code)]
const JR_F_CLIENT_RESPONSES: u32 = 1 << 5;

/// Sketch: the `requests` map of server.rs:144-151 completed from the device's ClientResponse runs of the batch just
/// taken (engine created with JR_F_CAPTURE_FSM | JR_F_CLIENT_RESPONSES, after jr_fsm_records_wait).  Address::Client
/// completes a local request; Address::Peer(n) is a proxied one the host relays to node n as Command::ClientResponse
/// (follower.rs:271-282).  `complete(group, token)` takes the oneshot out of `requests` and sends Ok(..) on it.
#[allow(dead_code)]
unsafe fn answer_clients(engine: *mut c_void, mut complete: impl FnMut(u32, u64), mut relay: impl FnMut(u32, u32, u64)) -> c_int {
    let mut runs: *const JrFsmRecord = std::ptr::null();
    let mut batch = [0u64; 8]; // jr_fsm_batch: n_records, n_dropped, n_instructions, node_offset[9], reserved
    let st = jr_fsm_responses(engine, &mut runs, batch.as_mut_ptr() as *mut c_void);
    if st != 0 && st != 4 {
        return st; // JR_E_CAPACITY (4): some requests stay unanswered (engine limits), the runs are still valid
    }
    for k in 0..batch[0] as usize {
        let r = &*runs.add(k);
        for i in 0..(r.hdr >> 8) as u64 {
            let token = r.tok0.wrapping_add(i.wrapping_mul(r.stride));
            match (r.addr >> 16) as u8 {
                A_PEER => relay(r.group, r.addr & 0xFFFF, token),
                _ => complete(r.group, token),
            }
        }
    }
    st
}

// Command discriminants, in the order of `enum Command` (src/raft/mod.rs:160-227)
const K_TICK: u8 = 0;
const K_VOTE_REQUEST: u8 = 2;
const K_VOTE_RESPONSE: u8 = 3;
const K_APPEND_ENTRIES: u8 = 4;
const K_APPEND_RESPONSE: u8 = 5;
const K_HEARTBEAT: u8 = 6;
const K_HEARTBEAT_RESPONSE: u8 = 7;
const K_CLIENT_REQUEST: u8 = 10;
const K_CLIENT_RESPONSE: u8 = 11;
// Address kinds (src/raft/rpc.rs:5-14)
const A_PEERS: u8 = 0;
const A_PEER: u8 = 1;
const A_LOCAL: u8 = 2;
const A_CLIENT: u8 = 3;

fn block_id(b: &BlockId) -> u64 {
    // BlockId is 8 big-endian bytes (chain.rs:63-66)
    let mut a = [0u8; 8];
    a.copy_from_slice(b.as_ref());
    u64::from_be_bytes(a)
}

/// Payload bytes and request ids never cross the FFI: blocks and requests carry 64-bit tokens.
#[derive(Default)]
pub struct Tokens {
    next: u64,
    payload: HashMap<u64, Vec<u8>>,
    request: HashMap<u64, (ClientRequestId, Address)>,
}

impl Tokens {
    fn intern(&mut self, data: Vec<u8>) -> u64 {
        self.next += 1;
        self.payload.insert(self.next, data);
        self.next
    }
}

fn addr(kind: u8, id: u32) -> Address {
    match kind {
        A_PEERS => Address::Peers,
        A_PEER => Address::Peer(id),
        A_LOCAL => Address::Local,
        _ => Address::Client,
    }
}

/// `Message` of the reference -> `jr_msg` to inject (the tcp_rx arm, server.rs:127-137).
fn encode(group: u32, me: NodeId, msg: &Message, tokens: &mut Tokens) -> JrMsg {
    let mut m = JrMsg { group, to_kind: A_PEER, to_id: me, ..Default::default() };
    if let Address::Peer(p) = msg.from {
        m.from_kind = A_PEER;
        m.from_id = p;
    }
    match &msg.command {
        Command::VoteRequest { term, candidate_id, last_term, head } => {
            m.kind = K_VOTE_REQUEST;
            m.term = *term;
            m.node_id = *candidate_id;
            m.last_term = *last_term;
            m.block = block_id(head);
        }
        Command::VoteResponse { term, from, granted } => {
            m.kind = K_VOTE_RESPONSE;
            m.term = *term;
            m.node_id = *from;
            m.flag = *granted as u8;
        }
        Command::AppendEntries { term, leader_id, blocks } => {
            m.kind = K_APPEND_ENTRIES;
            m.term = *term;
            m.node_id = *leader_id;
            m.n_blocks = blocks.len().min(JR_MAX_AE_BLOCKS) as u8; // MAX_INFLIGHT = 5, progress.rs:117
            for (i, b) in blocks.iter().take(JR_MAX_AE_BLOCKS).enumerate() {
                m.blocks[i] = JrBlock { id: block_id(&b.id), next: block_id(&b.next), data: tokens.intern(b.data.clone()) };
            }
        }
        Command::AppendResponse { node_id, term, head, success } => {
            m.kind = K_APPEND_RESPONSE;
            m.node_id = *node_id;
            m.term = *term;
            m.block = block_id(head);
            m.flag = *success as u8;
        }
        Command::Heartbeat { term, commit, leader_id } => {
            m.kind = K_HEARTBEAT;
            m.term = *term;
            m.block = block_id(commit);
            m.node_id = *leader_id;
        }
        Command::HeartbeatResponse { commit, has_committed } => {
            m.kind = K_HEARTBEAT_RESPONSE;
            m.block = block_id(commit);
            m.flag = *has_committed as u8;
        }
        _ => { /* Tick / Timeout / Noop never arrive over TCP; ClientRequest: see propose() */ }
    }
    m
}

/// `jr_msg` returned by the engine -> `Message` for tcp_tx (server.rs:141-142).
fn decode(me: NodeId, m: &JrMsg, tokens: &Tokens) -> Message {
    let id = |v: u64| BlockId::new(v);
    let command = match m.kind {
        K_VOTE_REQUEST => Command::VoteRequest { term: m.term, candidate_id: m.node_id, last_term: m.last_term, head: id(m.block) },
        K_VOTE_RESPONSE => Command::VoteResponse { term: m.term, from: m.node_id, granted: m.flag != 0 },
        K_APPEND_ENTRIES => Command::AppendEntries {
            term: m.term,
            leader_id: m.node_id,
            blocks: m.blocks[..m.n_blocks as usize]
                .iter()
                .map(|b| Block { id: id(b.id), next: id(b.next), data: tokens.payload.get(&b.data).cloned().unwrap_or_default() })
                .collect(),
        },
        K_APPEND_RESPONSE => Command::AppendResponse { node_id: m.node_id, term: m.term, head: id(m.block), success: m.flag != 0 },
        K_HEARTBEAT => Command::Heartbeat { term: m.term, commit: id(m.block), leader_id: m.node_id },
        K_HEARTBEAT_RESPONSE => Command::HeartbeatResponse { commit: id(m.block), has_committed: m.flag != 0 },
        _ => Command::Noop,
    };
    Message::new(Address::Peer(me), addr(m.to_kind, m.to_id), command)
}

pub struct StepOutput {
    pub messages: Vec<Message>,
    pub instructions: Vec<Instruction>,
    /// replicas of this engine that hold a sticky fault after the step (the reference would have left
    /// event_loop through `?` or a panic, server.rs:125-159)
    pub faulted: u64,
}

/// One hosted node (this process) of ONE Raft group on the GPU engine.  A multi-raft broker
/// would keep one engine for all its groups and index them by `group`.
pub struct GpuRaft {
    engine: *mut c_void,
    me: NodeId,
    group: u32,
    tokens: Tokens,
    out_msgs: Vec<JrMsg>,
    out_fsm: Vec<JrFsmInstr>,
}

impl GpuRaft {
    pub fn new(me: NodeId, n_nodes: u32, seed: u64) -> anyhow::Result<Self> {
        let mut cfg = JrConfig::default();
        unsafe { jr_config_default(&mut cfg, 1, n_nodes) };
        cfg.seed = seed;
        cfg.flags = JR_F_CAPTURE_MESSAGES | JR_F_CAPTURE_FSM;
        cfg.resident_mask = 1 << (me - 1); // this process hosts only `me` (RaftConfig::id, config.rs:23)
        let mut engine = std::ptr::null_mut();
        let st = unsafe { jr_engine_create(&cfg, &mut engine) };
        anyhow::ensure!(st == 0, "jr_engine_create failed: status {}", st);
        Ok(GpuRaft {
            engine,
            me,
            group: 0,
            tokens: Tokens::default(),
            out_msgs: vec![JrMsg::default(); 256],
            out_fsm: vec![JrFsmInstr::default(); 256],
        })
    }

    /// tcp_rx arm (server.rs:127-137): `raft.apply(msg.command)` NOW -- an inject-only step (no delivery, no Tick).
    pub fn on_peer_message(&mut self, now_ms: u64, msg: &Message) -> anyhow::Result<StepOutput> {
        let m = encode(self.group, self.me, msg, &mut self.tokens);
        self.step(now_ms, 0, &[m])
    }

    /// client arm (server.rs:156-160): `raft.apply(Command::ClientRequest(..))` NOW.
    pub fn propose(&mut self, now_ms: u64, id: ClientRequestId, proposal: Proposal) -> anyhow::Result<StepOutput> {
        let token = self.tokens.intern(proposal.get());
        self.tokens.request.insert(token, (id, Address::Client));
        let m = JrMsg { group: self.group, to_kind: A_PEER, to_id: self.me, from_kind: A_LOCAL, kind: K_CLIENT_REQUEST, token,
                        client_kind: A_CLIENT, ..Default::default() };
        self.step(now_ms, 0, &[m])
    }

    /// tick arm (server.rs:125): Command::Tick.  (With one resident node per engine there is no co-resident mail:
    /// DELIVER only matters when several nodes of the group live in this engine.)
    pub fn tick(&mut self, now_ms: u64) -> anyhow::Result<StepOutput> {
        self.step(now_ms, JR_STEP_DELIVER | JR_STEP_TICK, &[])
    }

    fn step(&mut self, now_ms: u64, flags: u32, inject: &[JrMsg]) -> anyhow::Result<StepOutput> {
        let mut args = JrStepArgs {
            now_ms,
            flags: flags | JR_STEP_REPORT_FAULTS,
            n_synth: 0,
            inject: inject.as_ptr(),
            n_inject: inject.len(),
            proposals: std::ptr::null(),
            out_msgs: self.out_msgs.as_mut_ptr(),
            cap_msgs: self.out_msgs.len(),
            n_msgs: 0,
            out_fsm: self.out_fsm.as_mut_ptr(),
            cap_fsm: self.out_fsm.len(),
            n_fsm: 0,
            n_faulted: 0,
        };
        let st = unsafe { jr_step(self.engine, &mut args) };
        anyhow::ensure!(st == 0, "jr_step failed: status {}", st);
        let messages = self.out_msgs[..args.n_msgs].iter().map(|m| decode(self.me, m, &self.tokens)).collect();
        let instructions = self.out_fsm[..args.n_fsm]
            .iter()
            .map(|f| {
                if f.kind == 0 {
                    Instruction::Apply {
                        block: Block {
                            id: BlockId::new(f.block.id),
                            next: BlockId::new(f.block.next),
                            data: self.tokens.payload.get(&f.block.data).cloned().unwrap_or_default(),
                        },
                    }
                } else {
                    let (id, _) = self.tokens.request[&f.block.data];
                    Instruction::Notify { id, client_address: addr(f.client_kind, f.client_id), block_id: BlockId::new(f.block.id) }
                }
            })
            .collect();
        Ok(StepOutput { messages, instructions, faulted: args.n_faulted })
    }
}

impl Drop for GpuRaft {
    fn drop(&mut self) {
        unsafe { jr_engine_destroy(self.engine) }
    }
}

// event_loop (src/raft/server.rs:103-165) with the engine in place of RaftHandle -- every arm applies its
// command at once, like the reference; `emit` forwards the outputs and turns a fault into the reference's Err:
//
//   let emit = |out: StepOutput| -> Result<()> {
//       if out.faulted != 0 { return Err(anyhow!("raft fault")); }                   // the reference's `?` / panic
//       for m in out.messages     { tcp_tx.send(m)?; }                                // server.rs:141-142
//       for i in out.instructions { fsm_tx.send(i)?; }                                // leader.rs:94,184; follower.rs:205
//       Ok(())
//   };
//   loop { tokio::select! {
//       _ = shutdown.wait()                       => break,
//       _ = step_interval.tick()                  => emit(raft.tick(now_ms())?)?,                       // server.rs:125
//       Some(msg) = tcp_rx.recv()                 => emit(raft.on_peer_message(now_ms(), &msg)?)?,      // server.rs:127-137
//       Some((proposal, res)) = client_rx.recv()  => { let id = Uuid::new_v4(); requests.insert(id, res);
//                                                      emit(raft.propose(now_ms(), id, proposal)?)?; }   // server.rs:156-160
//   } }
//
// A broker that hosts MANY groups keeps one engine for all of them and uses the batched calls instead
// (jr_run_tokens + jr_leader_table_async + jr_fsm_records_async / _wait / jr_fsm_fold): see INTEGRATION.md.
