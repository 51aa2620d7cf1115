// restated_raft.hpp -- C++ RESTATEMENT of josefine's src/raft state machine.
//
// TEST INFRASTRUCTURE ONLY.  This is the CPU oracle the CUDA engine is checked
// against and the "port" CPU baseline bench.py times.  It is NOT josefine: the
// reference is a Rust crate that cannot be built in this environment (no
// cargo/rustc).  It was written from reading the reference, function by
// function; every function cites the file:line it follows (paths relative to
// the reference checkout).  Only tests/, __graft_entry__.smoke() and bench.py's
// cpu_baseline / --impl reference legs may use anything under oracle/.
//
// Parity status: the reference's own known-answer tests (single voter + Chain)
// are ported in tests/test_oracle_kat.py and pin this file for those paths.
// Multi-replica behaviour is NOT pinned by any reference test ("parity
// unpinned", SURVEY.md section 8c); there the oracle is cross-checked by a
// second, independently written restatement (oracle/restated_raft.py).
//
// Deviations D1..D6 are the ones declared in include/josefine_raft_abi.h.
#pragma once
#include <cstdint>
#include <map>
#include <optional>
#include <vector>

#include "../include/josefine_raft_abi.h"

namespace restated {

using NodeId = uint32_t;   // mod.rs:136
using Term = uint64_t;     // mod.rs:139
using BlockId = uint64_t;  // chain.rs:29-67: 8-byte big-endian, so byte order == numeric order

struct Fault {
  int code;
};

// ---- rpc.rs:5-14 -----------------------------------------------------------
struct Address {
  uint8_t kind = JR_ADDR_PEERS;
  NodeId id = 0;
  static Address peers() { return {JR_ADDR_PEERS, 0}; }
  static Address peer(NodeId n) { return {JR_ADDR_PEER, n}; }
  static Address client() { return {JR_ADDR_CLIENT, 0}; }
  bool operator==(const Address& o) const { return kind == o.kind && id == o.id; }
};

// ---- chain.rs:86-91 ----------------------------------------------------------
struct Block {
  BlockId id = 0;
  BlockId next = 0;
  uint64_t data = 0;  // D5: payload token
};

// ---- mod.rs:145-150 ----------------------------------------------------------
struct ClientRequest {
  uint64_t id = 0;  // D5: Uuid -> token; the proposal payload is the same token
  Address address;
};

// ---- mod.rs:160-227 ----------------------------------------------------------
struct Command {
  uint8_t kind = JR_CMD_NOOP;
  Term term = 0;
  NodeId node_id = 0;  // candidate_id / from / leader_id / node_id
  Term last_term = 0;
  BlockId block = 0;   // head / commit
  bool flag = false;   // granted / success / has_committed
  std::vector<Block> blocks;
  ClientRequest req;   // ClientRequest / ClientResponse id
};

// ---- rpc.rs:17-21 ------------------------------------------------------------
struct Message {
  Address from, to;
  Command command;
};

// ---- fsm.rs:19-29 ------------------------------------------------------------
struct Instruction {
  uint8_t kind = JR_FSM_APPLY;
  Block block;          // Apply
  uint64_t req_id = 0;  // Notify
  Address client_address;
  BlockId block_id = 0;
};

// ---- chain.rs:99-253 ---------------------------------------------------------
// sled is modelled as an ordered map keyed by the 8-byte big-endian id.  The
// "commit" key (chain.rs:198) lives in the same sled tree and sorts after every
// block id below 0x63 << 56; `commit_key_` records whether it exists.
class Chain {
 public:
  Chain(uint64_t capacity, bool strict_commit_key);          // chain.rs:117-153, fresh data directory
  // chain.rs:117-137 over an existing data directory: the persisted blocks and "commit" value
  Chain(uint64_t capacity, bool strict_commit_key, const std::vector<Block>& persisted, uint64_t commit, bool commit_key,
        uint64_t floor);
  void truncate(BlockId floor);                              // deviation D7: keys below `floor` leave the tree
  void shift_ids(uint64_t k);                                // test-only (jro_shift_ids): ids >= floor move up by k
  BlockId floor() const { return floor_; }
  bool has(BlockId id) const;                                // chain.rs:155-157
  BlockId append(uint64_t data);                             // chain.rs:160-175
  void extend(const Block& b);                               // chain.rs:178-192
  BlockId commit(BlockId id);                                // chain.rs:195-205
  // chain.rs:208-228 with the three bound shapes the callers use.
  std::vector<Block> range_half_open(BlockId lo, BlockId hi) const;   // lo..hi
  std::vector<Block> range_inclusive(BlockId lo, BlockId hi) const;   // lo..=hi
  // lo.. then .skip(skip).take(take): the only unbounded ranges (leader.rs:135,152-157)
  std::vector<Block> range_from_skip_take(BlockId lo, size_t skip, size_t take) const;
  void compact();                                            // chain.rs:239-253
  BlockId get_head() const { return head_; }                 // chain.rs:230-232
  BlockId get_commit() const { return commit_; }             // chain.rs:234-236
  uint64_t id_gen() const { return id_gen_; }
  const std::map<BlockId, Block>& blocks() const { return db_; }

 private:
  void check_capacity(BlockId id) const;
  std::map<BlockId, Block> db_;
  bool commit_key_ = false;
  bool strict_ = false;
  uint64_t capacity_;
  BlockId floor_ = 0;
  uint64_t id_gen_ = 0;
  BlockId commit_ = 0;
  BlockId head_ = 0;
};

// ---- election.rs:6-74 --------------------------------------------------------
enum class ElectionStatus { Elected, Voting, Defeated };
class Election {
 public:
  explicit Election(std::vector<NodeId> voters) : voter_ids_(std::move(voters)) {}
  void reset() { votes_.clear(); }                                  // election.rs:29-31
  void vote(NodeId id, bool v) { votes_[id] = v; }                  // election.rs:33-35 (last write wins)
  ElectionStatus status() const;                                    // election.rs:37-57
  size_t quorum_size() const;                                       // election.rs:66-73
  const std::map<NodeId, bool>& votes() const { return votes_; }

 private:
  std::vector<NodeId> voter_ids_;
  std::map<NodeId, bool> votes_;
};

// ---- progress.rs:10-232 ------------------------------------------------------
struct NodeProgress {
  enum Kind { Probe, Replicate, Snapshot } kind = Probe;
  NodeId node_id = 0;
  BlockId head = 0;
  bool active = false;  // carried along, never read for Probe/Replicate (progress.rs:164-166,216-218)
  void advance(BlockId id);   // progress.rs:76-94 + 133-140
  bool is_active() const;     // progress.rs:96-102
};
class ReplicationProgress {
 public:
  explicit ReplicationProgress(const std::vector<NodeId>& nodes);  // progress.rs:15-23
  NodeProgress* get_mut(NodeId id);                                // progress.rs:29-31
  std::map<NodeId, NodeProgress>& all_mut() { return progress_; }  // test-only (jro_shift_ids)
  void advance(NodeId id, BlockId block);                          // progress.rs:42-46
  BlockId committed_index() const;                                 // progress.rs:48-60
  const std::map<NodeId, NodeProgress>& all() const { return progress_; }

 private:
  std::map<NodeId, NodeProgress> progress_;
};

struct NodeConfig {
  NodeId id = 1;
  std::vector<NodeId> peers;  // RaftConfig::nodes, config.rs:28 (ids only; ascending)
  uint64_t seed = 0;
  uint64_t group = 0;         // global group id (D2 key)
  uint32_t election_min_ms = 500, election_max_ms = 1000, heartbeat_ms = 100;
  uint64_t chain_capacity = 1u << 20;
  bool strict_commit_key = false;
};

// ---- mod.rs:271-341, roles folded into one object ---------------------------
class Node {
 public:
  explicit Node(const NodeConfig& cfg);  // follower.rs:68-95
  Node(const NodeConfig& cfg, Chain persisted, uint64_t now);  // the same over an existing data directory, at time `now`
  // Apply::apply (mod.rs:471-479).  `now` replaces Instant::now() (D1).  Output
  // is appended to rpc / fsm (rpc_tx / fsm_tx, mod.rs:338-340).  A reference
  // panic or Err sets fault() and the node ignores everything afterwards (D3).
  void apply(const Command& cmd, uint64_t now);

  // inspection
  int role() const { return role_; }
  int fault() const { return fault_; }
  const NodeConfig& config() const { return cfg_; }
  Term current_term = 0;                       // State, mod.rs:276
  std::optional<NodeId> voted_for;             // mod.rs:278
  uint64_t election_time = 0;                  // mod.rs:280 (always Some after init)
  uint32_t election_timeout = 0;               // mod.rs:282
  uint32_t rng_draws = 0;                      // D2
  std::optional<NodeId> leader_id;             // Follower, follower.rs:21
  std::vector<ClientRequest> queued_reqs;      // Follower/Candidate, follower.rs:23, candidate.rs:20
  std::optional<Election> election;            // Candidate, candidate.rs:19
  std::optional<ReplicationProgress> progress; // Leader, leader.rs:25
  uint64_t heartbeat_time = 0;                 // Leader, leader.rs:27
  Chain chain;
  std::vector<Message> rpc;
  std::vector<Instruction> fsm;
  bool alive = true;

 private:
  void dispatch(const Command& cmd);
  // mod.rs
  bool needs_election() const;                        // mod.rs:352-357
  void set_term(Term t);                              // mod.rs:360-365 + Role::term impls
  void send(Address to, Command cmd);                 // mod.rs:390-394
  void send_all(Command cmd);                         // mod.rs:396-400
  // follower.rs
  void follower_apply(const Command& cmd);            // follower.rs:38-63
  bool can_vote(Term last_term, BlockId head) const;  // follower.rs:97-101
  void set_election_timeout();                        // follower.rs:103-113
  void follower_append_entries(const Command& c);     // follower.rs:130-176
  void follower_heartbeat(const Command& c);          // follower.rs:178-217
  void follower_vote_request(const Command& c);       // follower.rs:219-246
  void follower_timeout();                            // follower.rs:248-256
  void follower_client_request(ClientRequest req);    // follower.rs:258-269
  void become_candidate();                            // follower.rs:285-304
  // candidate.rs
  void candidate_apply(const Command& cmd);           // candidate.rs:170-196
  void seek_election();                               // candidate.rs:24-45
  void candidate_tick();                              // candidate.rs:48-68
  void candidate_vote_request(const Command& c);      // candidate.rs:71-88
  void candidate_vote_response(const Command& c);     // candidate.rs:91-113
  void candidate_append_entries(const Command& c);    // candidate.rs:116-134
  void candidate_heartbeat(const Command& c);         // candidate.rs:137-157
  void candidate_to_follower();                       // candidate.rs:198-214
  void candidate_to_leader();                         // candidate.rs:216-238
  // leader.rs
  void leader_apply(const Command& cmd);              // leader.rs:248-266
  void heartbeat();                                   // leader.rs:44-51
  void leader_commit();                               // leader.rs:87-99
  void replicate();                                   // leader.rs:124-174
  void leader_client_request(const ClientRequest& r); // leader.rs:177-197
  void leader_tick();                                 // leader.rs:234-245

  NodeConfig cfg_;
  int role_ = JR_ROLE_FOLLOWER;
  int fault_ = JR_FAULT_NONE;
  uint64_t now_ = 0;
};

uint64_t mix64(uint64_t x);
uint32_t election_timeout_draw(uint64_t seed, uint64_t group, uint32_t node, uint32_t draw,
                               uint32_t min_ms, uint32_t max_ms);

}  // namespace restated
