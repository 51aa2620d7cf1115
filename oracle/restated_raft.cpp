// restated_raft.cpp -- C++ RESTATEMENT of josefine's src/raft (see restated_raft.hpp).
// TEST INFRASTRUCTURE ONLY; not josefine, not shipped on the product path.
#include "restated_raft.hpp"

#include <algorithm>

namespace restated {

// ---- D2: counter-based election timeout (normative text in the ABI header) ----
uint64_t mix64(uint64_t x) {
  x += 0x9e3779b97f4a7c15ull;
  x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ull;
  x = (x ^ (x >> 27)) * 0x94d049bb133111ebull;
  return x ^ (x >> 31);
}

uint32_t election_timeout_draw(uint64_t seed, uint64_t group, uint32_t node, uint32_t draw,
                               uint32_t min_ms, uint32_t max_ms) {
  uint64_t x = mix64(seed ^ 0x6a09e667f3bcc908ull);
  x = mix64(x + group);
  x = mix64(x + (((uint64_t)node << 32) | draw));
  uint64_t span = (uint64_t)(max_ms - min_ms);
  return min_ms + (uint32_t)(((x >> 32) * span) >> 32);
}

// =============================== Chain =========================================

// chain.rs:117-153.  A fresh sled has no "commit" key, so commit = 0 and init()
// writes the genesis block 0 -> 0 with the first generated id.
Chain::Chain(uint64_t capacity, bool strict) : strict_(strict), capacity_(capacity) {
  uint64_t id = id_gen_++;  // chain.rs:140-141: asserts this is 0
  db_[id] = Block{id, id, 0};
}

// chain.rs:117-137 reopening a data directory: id_gen = head = commit = the persisted "commit" value (0 if the key
// is missing); commit == 0 runs init() again, which (re)writes the genesis block and leaves id_gen at 1.
Chain::Chain(uint64_t capacity, bool strict, const std::vector<Block>& persisted, uint64_t commit, bool commit_key,
             uint64_t floor)
    : commit_key_(commit_key), strict_(strict), capacity_(capacity), floor_(floor), id_gen_(commit), commit_(commit),
      head_(commit) {
  for (const Block& b : persisted) db_[b.id] = b;
  if (commit == 0) {
    uint64_t id = id_gen_++;
    if (floor_ == 0) db_[id] = Block{id, id, 0};
  }
}

void Chain::check_capacity(BlockId id) const {
  if (id < floor_ || id - floor_ >= capacity_ || id >= JR_BLOCK_ID_LIMIT) throw Fault{JR_FAULT_ENGINE_CHAIN_CAPACITY};  // D4, D7
}

void Chain::shift_ids(uint64_t k) {  // test-only: f(v) = v + k for v >= floor, v below it unchanged
  auto f = [&](BlockId v) { return v >= floor_ ? v + k : v; };
  std::map<BlockId, Block> db;
  for (auto& kv : db_) db[f(kv.first)] = Block{f(kv.second.id), f(kv.second.next), kv.second.data};
  db_.swap(db);
  id_gen_ = f(id_gen_);
  commit_ = f(commit_);
  head_ = f(head_);
  floor_ += k;
}

void Chain::truncate(BlockId floor) {  // D7
  if (floor <= floor_) return;
  db_.erase(db_.begin(), db_.lower_bound(floor));
  floor_ = floor;
}

bool Chain::has(BlockId id) const { return db_.count(id) != 0; }  // chain.rs:155-157

// chain.rs:160-175.  fetch_add happens before the assert, so a failed append
// still consumes an id.
BlockId Chain::append(uint64_t data) {
  uint64_t id = id_gen_++;
  if (!(id > head_)) throw Fault{JR_FAULT_APPEND_ID_NOT_GT_HEAD};  // chain.rs:163
  check_capacity(id);
  db_[id] = Block{id, head_, data};
  head_ = id;
  return id;
}

// chain.rs:178-192.  Overwrites an existing id; head follows the block
// unconditionally; id_gen is not advanced.
void Chain::extend(const Block& b) {
  if (!has(b.next)) throw Fault{JR_FAULT_EXTEND_PARENT_MISSING};  // chain.rs:180-185
  check_capacity(b.id);
  db_[b.id] = b;
  head_ = b.id;
}

// chain.rs:195-205.
BlockId Chain::commit(BlockId id) {
  if (!has(id)) throw Fault{JR_FAULT_COMMIT_BLOCK_MISSING};  // chain.rs:200-202
  commit_key_ = true;                                        // db.insert("commit", ..), chain.rs:198
  commit_ = id;
  return id;
}

std::vector<Block> Chain::range_half_open(BlockId lo, BlockId hi) const {
  std::vector<Block> out;
  for (auto it = db_.lower_bound(lo); it != db_.end() && it->first < hi; ++it) out.push_back(it->second);
  return out;
}

std::vector<Block> Chain::range_inclusive(BlockId lo, BlockId hi) const {
  std::vector<Block> out;
  for (auto it = db_.lower_bound(lo); it != db_.end() && it->first <= hi; ++it) out.push_back(it->second);
  return out;
}

// db.range(lo..) is unbounded above, so after the last block it yields the
// "commit" entry, whose 8-byte value is not a bincode Block: the map closure at
// chain.rs:221-226 panics.  skip(n).take(m) pulls n+m items before stopping
// (nth(1) == skip(1).take(1)), so the panic happens exactly when fewer than n+m
// blocks remain and the key exists.  Only with JR_F_SLED_COMMIT_KEY_STRICT (D6).
std::vector<Block> Chain::range_from_skip_take(BlockId lo, size_t skip, size_t take) const {
  std::vector<Block> out;
  size_t pulled = 0;
  auto it = db_.lower_bound(lo);
  while (pulled < skip + take) {
    if (it == db_.end()) {
      if (strict_ && commit_key_) throw Fault{JR_FAULT_RANGE_COMMIT_KEY};
      break;
    }
    if (pulled >= skip) out.push_back(it->second);
    ++pulled;
    ++it;
  }
  return out;
}

// chain.rs:239-253: walk ids in [0, commit) from the top; the first is kept;
// afterwards a block is removed when its id is not the `next` of the block
// visited before it -- and the expectation moves to the visited block's own
// `next` whether or not it was removed.
void Chain::compact() {
  std::optional<BlockId> next_id;
  std::vector<Block> walk = range_half_open(0, commit_);
  for (auto it = walk.rbegin(); it != walk.rend(); ++it) {
    if (next_id.has_value() && it->id != *next_id) db_.erase(it->id);
    next_id = it->next;
  }
}

// =============================== Election ======================================

size_t Election::quorum_size() const {  // election.rs:66-73
  if (voter_ids_.size() == 1) return 0;
  return voter_ids_.size() / 2 + 1;
}

ElectionStatus Election::status() const {  // election.rs:37-57
  size_t votes = 0, total = 0;
  for (auto& kv : votes_) {
    if (kv.second) ++votes;
    ++total;
  }
  if (votes >= quorum_size()) return ElectionStatus::Elected;
  if (total - votes == quorum_size()) return ElectionStatus::Defeated;  // exact equality
  return ElectionStatus::Voting;
}

// =============================== Progress ======================================

void NodeProgress::advance(BlockId id) {  // progress.rs:76-94,133-140
  bool incremented = false;
  if (head < id) {
    head = id;
    incremented = true;
  }
  switch (kind) {
    case Probe: kind = incremented ? Replicate : Probe; break;
    case Replicate: kind = incremented ? Replicate : Probe; break;
    default: throw Fault{JR_FAULT_PROGRESS_UNKNOWN_NODE};  // progress.rs:92 panic!(), unreachable
  }
}

bool NodeProgress::is_active() const {  // progress.rs:96-102,164-166,216-218
  // Probe: !paused, never paused.  Replicate: capacity(>=5) > len(0).  Always true.
  return kind == Snapshot ? active : true;
}

ReplicationProgress::ReplicationProgress(const std::vector<NodeId>& nodes) {  // progress.rs:15-23
  for (NodeId n : nodes) {
    NodeProgress p;
    p.node_id = n;
    progress_[n] = p;
  }
}

NodeProgress* ReplicationProgress::get_mut(NodeId id) {
  auto it = progress_.find(id);
  return it == progress_.end() ? nullptr : &it->second;
}

void ReplicationProgress::advance(NodeId id, BlockId block) {  // progress.rs:42-46
  auto it = progress_.find(id);
  if (it == progress_.end()) throw Fault{JR_FAULT_PROGRESS_UNKNOWN_NODE};
  it->second.advance(block);
}

BlockId ReplicationProgress::committed_index() const {  // progress.rs:48-60
  std::vector<BlockId> idx;
  for (auto& kv : progress_) idx.push_back(kv.second.head);
  std::sort(idx.begin(), idx.end(), [](BlockId a, BlockId b) { return a > b; });
  return idx[idx.size() / 2];
}

// ================================= Node ========================================

Node::Node(const NodeConfig& cfg)  // follower.rs:68-95
    : chain(cfg.chain_capacity, cfg.strict_commit_key), cfg_(cfg) {
  // init(): set_election_timeout at time 0 of the logical clock
  now_ = 0;
  set_election_timeout();
}

Node::Node(const NodeConfig& cfg, Chain persisted, uint64_t now) : chain(std::move(persisted)), cfg_(cfg) {
  now_ = now;
  set_election_timeout();
}

void Node::apply(const Command& cmd, uint64_t now) {
  if (!alive || fault_ != JR_FAULT_NONE) return;
  now_ = now;
  try {
    dispatch(cmd);
  } catch (const Fault& f) {
    fault_ = f.code;  // D3: panic / Err ends the node
  }
}

void Node::dispatch(const Command& cmd) {  // mod.rs:471-479
  switch (role_) {
    case JR_ROLE_FOLLOWER: follower_apply(cmd); break;
    case JR_ROLE_CANDIDATE: candidate_apply(cmd); break;
    default: leader_apply(cmd); break;
  }
}

bool Node::needs_election() const {  // mod.rs:352-357; Instant::elapsed saturates
  uint64_t elapsed = now_ >= election_time ? now_ - election_time : 0;
  return elapsed > election_timeout;
}

void Node::set_term(Term t) {  // mod.rs:360-365
  voted_for.reset();
  current_term = t;
  switch (role_) {
    case JR_ROLE_FOLLOWER: leader_id.reset(); break;   // follower.rs:27-29
    case JR_ROLE_CANDIDATE: election->reset(); break;  // candidate.rs:161-163
    default: throw Fault{JR_FAULT_LEADER_TERM_UNIMPLEMENTED};  // leader.rs:33-35
  }
}

void Node::send(Address to, Command cmd) {  // mod.rs:390-394
  rpc.push_back(Message{Address::peer(cfg_.id), to, std::move(cmd)});
}

void Node::send_all(Command cmd) {  // mod.rs:396-400
  rpc.push_back(Message{Address::peer(cfg_.id), Address::peers(), std::move(cmd)});
}

// ------------------------------- follower --------------------------------------

void Node::follower_apply(const Command& cmd) {  // follower.rs:38-63
  switch (cmd.kind) {
    case JR_CMD_TICK:  // follower.rs:121-128
      if (needs_election()) follower_apply(Command{JR_CMD_TIMEOUT});
      break;
    case JR_CMD_APPEND_ENTRIES: follower_append_entries(cmd); break;
    case JR_CMD_HEARTBEAT: follower_heartbeat(cmd); break;
    case JR_CMD_VOTE_REQUEST: follower_vote_request(cmd); break;
    case JR_CMD_TIMEOUT: follower_timeout(); break;
    case JR_CMD_CLIENT_REQUEST: follower_client_request(cmd.req); break;
    case JR_CMD_CLIENT_RESPONSE: {  // follower.rs:271-282 (proxied_reqs is bookkeeping only)
      Command c{JR_CMD_CLIENT_RESPONSE};
      c.req = cmd.req;
      send(Address::client(), c);
      break;
    }
    default: break;  // apply_self
  }
}

bool Node::can_vote(Term last_term, BlockId head) const {  // follower.rs:97-101
  return !(voted_for.has_value() || current_term > last_term || chain.get_commit() > head);
}

void Node::set_election_timeout() {  // follower.rs:103-113, D2
  election_timeout = election_timeout_draw(cfg_.seed, cfg_.group, cfg_.id, rng_draws++,
                                           cfg_.election_min_ms, cfg_.election_max_ms);
  election_time = now_;
}

void Node::follower_append_entries(const Command& c) {  // follower.rs:130-176
  NodeId leader = c.node_id;
  if (!voted_for.has_value() && c.term >= current_term) {
    set_term(c.term);
    election_time = now_;  // timer restarted, timeout value kept (follower.rs:141)
    leader_id = leader;
    voted_for = leader;
  }
  if (voted_for.has_value()) {
    if (*voted_for != leader && c.term < current_term) throw Fault{JR_FAULT_AE_STALE_LEADER};
  }
  if (!c.blocks.empty()) {
    for (const Block& b : c.blocks) chain.extend(b);  // Err -> `?` -> server stops
    Command r{JR_CMD_APPEND_RESPONSE};
    r.node_id = cfg_.id;
    r.term = current_term;
    r.block = chain.get_head();
    r.flag = true;
    send(Address::peer(leader), r);
  }
}

void Node::follower_heartbeat(const Command& c) {  // follower.rs:178-217
  NodeId leader = c.node_id;
  set_election_timeout();
  set_term(c.term);  // unconditional, even for a lower term
  leader_id = leader;
  voted_for = leader;
  std::vector<ClientRequest> q;
  q.swap(queued_reqs);
  for (auto& req : q) {  // follower.rs:190-197
    Command f{JR_CMD_CLIENT_REQUEST};
    f.req = req;
    send(Address::peer(leader), f);
  }
  bool has = chain.has(c.block);
  if (has && c.block > chain.get_commit()) {
    BlockId prev = chain.get_commit();
    chain.commit(c.block);
    for (const Block& b : chain.range_half_open(prev, c.block)) {  // prev..commit, follower.rs:204
      Instruction i;
      i.kind = JR_FSM_APPLY;
      i.block = b;
      fsm.push_back(i);
    }
  }
  Command r{JR_CMD_HEARTBEAT_RESPONSE};
  r.block = chain.get_commit();
  r.flag = has;
  send(Address::peer(leader), r);
}

void Node::follower_vote_request(const Command& c) {  // follower.rs:219-246 (request term ignored)
  Command r{JR_CMD_VOTE_RESPONSE};
  r.term = current_term;
  r.node_id = cfg_.id;
  r.flag = can_vote(c.last_term, c.block);
  send(Address::peer(c.node_id), r);
  if (r.flag) voted_for = c.node_id;
}

void Node::follower_timeout() {  // follower.rs:248-256
  if (!voted_for.has_value()) {
    set_election_timeout();
    become_candidate();
    seek_election();
  }
}

void Node::follower_client_request(ClientRequest req) {  // follower.rs:258-269
  req.address = Address::peer(cfg_.id);
  if (leader_id.has_value()) {
    Command f{JR_CMD_CLIENT_REQUEST};
    f.req = req;
    send(Address::peer(*leader_id), f);
  } else {
    if (queued_reqs.size() >= JR_CLIENT_QUEUE_CAP) throw Fault{JR_FAULT_ENGINE_QUEUE_OVERFLOW};
    queued_reqs.push_back(req);
  }
}

void Node::become_candidate() {  // follower.rs:285-304: fresh Election, queued_reqs NOT carried
  std::vector<NodeId> voters = cfg_.peers;
  voters.push_back(cfg_.id);
  election.emplace(voters);
  queued_reqs.clear();
  leader_id.reset();
  role_ = JR_ROLE_CANDIDATE;
}

// ------------------------------- candidate -------------------------------------

void Node::candidate_apply(const Command& cmd) {  // candidate.rs:170-196
  switch (cmd.kind) {
    case JR_CMD_TICK: candidate_tick(); break;
    case JR_CMD_VOTE_REQUEST: candidate_vote_request(cmd); break;
    case JR_CMD_VOTE_RESPONSE: candidate_vote_response(cmd); break;
    case JR_CMD_APPEND_ENTRIES: candidate_append_entries(cmd); break;
    case JR_CMD_HEARTBEAT: candidate_heartbeat(cmd); break;
    case JR_CMD_CLIENT_REQUEST:
      if (queued_reqs.size() >= JR_CLIENT_QUEUE_CAP) throw Fault{JR_FAULT_ENGINE_QUEUE_OVERFLOW};
      queued_reqs.push_back(cmd.req);
      break;
    default: break;
  }
}

void Node::seek_election() {  // candidate.rs:24-45
  voted_for = cfg_.id;
  current_term += 1;
  Term term = current_term;
  for (size_t i = 0; i < cfg_.peers.size(); ++i) {  // one broadcast PER PEER: N-1 copies reach each peer
    Command v{JR_CMD_VOTE_REQUEST};
    v.term = term;
    v.node_id = cfg_.id;
    v.last_term = term;
    v.block = chain.get_head();
    send_all(v);
  }
  Command self{JR_CMD_VOTE_RESPONSE};
  self.node_id = cfg_.id;
  self.term = term;
  self.flag = true;
  candidate_apply(self);
}

void Node::candidate_tick() {  // candidate.rs:48-68
  if (!needs_election()) return;
  switch (election->status()) {
    case ElectionStatus::Voting:
    case ElectionStatus::Defeated:
      voted_for.reset();
      candidate_to_follower();
      follower_apply(Command{JR_CMD_TIMEOUT});
      break;
    default: throw Fault{JR_FAULT_CANDIDATE_TICK_ELECTED};  // candidate.rs:63
  }
}

void Node::candidate_vote_request(const Command& c) {  // candidate.rs:71-88
  if (c.term > current_term) {
    set_term(c.term);
    candidate_to_follower();  // no reply, no vote
    return;
  }
  Command r{JR_CMD_VOTE_RESPONSE};
  r.node_id = cfg_.id;
  r.term = current_term;
  r.flag = false;
  send(Address::peer(c.node_id), r);
}

void Node::candidate_vote_response(const Command& c) {  // candidate.rs:91-113 (response term ignored)
  election->vote(c.node_id, c.flag);
  switch (election->status()) {
    case ElectionStatus::Elected:  // elect(): transition first, then heartbeat
      candidate_to_leader();
      heartbeat();
      break;
    case ElectionStatus::Voting: break;
    case ElectionStatus::Defeated:
      voted_for.reset();
      candidate_to_follower();
      break;
  }
}

void Node::candidate_append_entries(const Command& c) {  // candidate.rs:116-134 (blocks dropped)
  if (c.term >= current_term) candidate_to_follower();
}

void Node::candidate_heartbeat(const Command& c) {  // candidate.rs:137-157
  bool has = chain.has(c.block);
  BlockId commit = chain.get_commit();
  set_term(c.term);
  voted_for = c.node_id;
  candidate_to_follower();
  Command r{JR_CMD_HEARTBEAT_RESPONSE};
  r.block = commit;
  r.flag = has;
  send(Address::peer(c.node_id), r);
}

void Node::candidate_to_follower() {  // candidate.rs:198-214: leader_id None, queued_reqs carried
  election.reset();
  leader_id.reset();
  role_ = JR_ROLE_FOLLOWER;
}

void Node::candidate_to_leader() {  // candidate.rs:216-238 (on_transition is a no-op, leader.rs:53-76)
  std::vector<NodeId> nodes = cfg_.peers;
  nodes.push_back(cfg_.id);
  progress.emplace(nodes);
  heartbeat_time = now_;
  election.reset();
  queued_reqs.clear();  // Leader has no queue
  role_ = JR_ROLE_LEADER;
}

// -------------------------------- leader ----------------------------------------

void Node::leader_apply(const Command& cmd) {  // leader.rs:248-266
  switch (cmd.kind) {
    case JR_CMD_TICK: leader_tick(); break;
    case JR_CMD_HEARTBEAT_RESPONSE:  // leader.rs:222-231
      if (!cmd.flag && cmd.block > 0) replicate();
      break;
    case JR_CMD_APPEND_RESPONSE:  // leader.rs:211-219 (term and success ignored)
      progress->advance(cmd.node_id, cmd.block);
      leader_commit();
      break;
    case JR_CMD_APPEND_ENTRIES:  // leader.rs:200-208
      if (cmd.term > current_term) set_term(cmd.term);  // -> unimplemented!()
      break;
    case JR_CMD_CLIENT_REQUEST: leader_client_request(cmd.req); break;
    default: break;
  }
}

void Node::heartbeat() {  // leader.rs:44-51
  Command h{JR_CMD_HEARTBEAT};
  h.term = current_term;
  h.block = chain.get_commit();
  h.node_id = cfg_.id;
  send_all(h);
}

void Node::leader_commit() {  // leader.rs:87-99
  BlockId q = progress->committed_index();
  if (q > chain.get_commit()) {
    BlockId prev = chain.get_commit();
    BlockId nw = chain.commit(q);
    bool first = true;
    for (const Block& b : chain.range_inclusive(prev, nw)) {  // (prev..=new).skip(1)
      if (first) {
        first = false;
        continue;
      }
      Instruction i;
      i.kind = JR_FSM_APPLY;
      i.block = b;
      fsm.push_back(i);
    }
  }
}

void Node::replicate() {  // leader.rs:124-174; config.nodes = peers only
  for (NodeId peer : cfg_.peers) {
    NodeProgress* p = progress->get_mut(peer);
    if (!p || !p->is_active()) continue;
    Command ae{JR_CMD_APPEND_ENTRIES};
    ae.term = current_term;
    ae.node_id = cfg_.id;
    if (p->kind == NodeProgress::Probe) {
      ae.blocks = chain.range_from_skip_take(p->head, 1, 1);  // range(head..).nth(1), may be empty
    } else if (p->kind == NodeProgress::Replicate) {
      ae.blocks = chain.range_from_skip_take(p->head, 1, JR_MAX_AE_BLOCKS);  // skip(1).take(5)
    } else {
      continue;
    }
    rpc.push_back(Message{Address::peer(cfg_.id), Address::peer(peer), ae});
  }
}

void Node::leader_client_request(const ClientRequest& req) {  // leader.rs:177-197
  Term term = current_term;
  BlockId block_id = chain.append(req.id);
  Instruction n;
  n.kind = JR_FSM_NOTIFY;
  n.req_id = req.id;
  n.block_id = block_id;
  n.client_address = req.address;
  fsm.push_back(n);
  Command self{JR_CMD_APPEND_RESPONSE};
  self.node_id = cfg_.id;
  self.term = term;
  self.flag = true;
  self.block = chain.get_head();
  leader_apply(self);
}

void Node::leader_tick() {  // leader.rs:234-245 (write_state's file dump -> jr_leader_table)
  uint64_t elapsed = now_ >= heartbeat_time ? now_ - heartbeat_time : 0;
  if (elapsed > cfg_.heartbeat_ms) {  // leader.rs:78-80
    heartbeat();
    heartbeat_time = now_;
  }
  replicate();
}

}  // namespace restated
