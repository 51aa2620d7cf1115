// restated_cluster.cpp -- batched harness + C API (jro_*) around the C++
// RESTATEMENT of josefine's src/raft.  TEST INFRASTRUCTURE ONLY.
//
// The harness applies the synthetic schedule documented at jr_step_args in
// include/josefine_raft_abi.h to G independent groups of R restated nodes, so
// the CUDA engine (jr_*) and this oracle (jro_*) can be driven by the same
// calls and compared bit for bit.  The schedule is ours; the per-command
// behaviour is the reference's (restated_raft.cpp).
#include <algorithm>
#include <cstring>
#include <memory>
#include <string>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <thread>

#include "restated_raft.hpp"

using namespace restated;

namespace {

inline uint64_t fold(uint64_t h, uint64_t w) { return mix64(h ^ w); }

jr_msg to_abi(const Message& m, uint32_t group) {
  jr_msg o;
  std::memset(&o, 0, sizeof o);
  o.group = group;
  o.from_kind = m.from.kind;
  o.from_id = m.from.id;
  o.to_kind = m.to.kind;
  o.to_id = m.to.id;
  const Command& c = m.command;
  o.kind = c.kind;
  switch (c.kind) {
    case JR_CMD_VOTE_REQUEST:
      o.term = c.term; o.node_id = c.node_id; o.last_term = c.last_term; o.block = c.block; break;
    case JR_CMD_VOTE_RESPONSE:
      o.term = c.term; o.node_id = c.node_id; o.flag = c.flag; break;
    case JR_CMD_APPEND_ENTRIES:
      o.term = c.term; o.node_id = c.node_id; o.n_blocks = (uint8_t)c.blocks.size();
      for (size_t i = 0; i < c.blocks.size() && i < JR_MAX_AE_BLOCKS; ++i)
        o.blocks[i] = jr_block{c.blocks[i].id, c.blocks[i].next, c.blocks[i].data};
      break;
    case JR_CMD_APPEND_RESPONSE:
      o.node_id = c.node_id; o.term = c.term; o.block = c.block; o.flag = c.flag; break;
    case JR_CMD_HEARTBEAT:
      o.term = c.term; o.block = c.block; o.node_id = c.node_id; break;
    case JR_CMD_HEARTBEAT_RESPONSE:
      o.block = c.block; o.flag = c.flag; break;
    case JR_CMD_CLIENT_REQUEST:
      o.token = c.req.id; o.client_kind = c.req.address.kind; o.client_id = c.req.address.id; break;
    case JR_CMD_CLIENT_RESPONSE:
      o.token = c.req.id; break;
    default: break;
  }
  return o;
}

Command from_abi(const jr_msg& m) {
  Command c;
  c.kind = m.kind;
  c.term = m.term;
  c.node_id = m.node_id;
  c.last_term = m.last_term;
  c.block = m.block;
  c.flag = m.flag != 0;
  for (unsigned i = 0; i < m.n_blocks && i < JR_MAX_AE_BLOCKS; ++i)
    c.blocks.push_back(Block{m.blocks[i].id, m.blocks[i].next, m.blocks[i].data});
  c.req.id = m.token;
  c.req.address = Address{m.client_kind, m.client_id};
  return c;
}

// Normative stream digests (DESIGN.md "Digests").
uint64_t digest_msg(uint64_t d, const jr_msg& m) {
  d = fold(d, (uint64_t)m.kind | ((uint64_t)m.to_kind << 8) | ((uint64_t)(m.flag ? 1 : 0) << 16) |
                  ((uint64_t)m.n_blocks << 24) | ((uint64_t)m.to_id << 32));
  d = fold(d, m.node_id);
  d = fold(d, m.term);
  d = fold(d, m.last_term);
  d = fold(d, m.block);
  d = fold(d, m.token);
  d = fold(d, (uint64_t)m.client_kind | ((uint64_t)m.client_id << 8));
  for (unsigned i = 0; i < m.n_blocks; ++i) {
    d = fold(d, m.blocks[i].id);
    d = fold(d, m.blocks[i].next);
    d = fold(d, m.blocks[i].data);
  }
  return d;
}

jr_fsm_instr fsm_to_abi(const Instruction& i, uint32_t group, uint32_t node) {
  jr_fsm_instr o;
  std::memset(&o, 0, sizeof o);
  o.group = group;
  o.node = node;
  o.kind = i.kind;
  if (i.kind == JR_FSM_APPLY) {
    o.block = jr_block{i.block.id, i.block.next, i.block.data};
  } else {
    o.client_kind = i.client_address.kind;
    o.client_id = i.client_address.id;
    o.block = jr_block{i.block_id, 0, i.req_id};
  }
  return o;
}

uint64_t digest_fsm(uint64_t d, const jr_fsm_instr& f) {
  d = fold(d, (uint64_t)f.kind | ((uint64_t)f.client_kind << 8) | ((uint64_t)f.client_id << 32));
  d = fold(d, f.block.id);
  d = fold(d, f.block.next);
  d = fold(d, f.block.data);
  return d;
}

struct Replica {
  std::unique_ptr<Node> node;
  std::vector<Message> prev_out;  // mail emitted in the previous step
  uint64_t msg_digest = 0, fsm_digest = 0;
  uint64_t n_msgs = 0, n_fsm = 0;
  size_t fsm_digested = 0;  // prefix of node->fsm already folded into fsm_digest
};

}  // namespace

// Persistent workers: thread t always owns the same contiguous slice of groups, so
// its nodes' allocations stay in its own malloc arena (spawning threads per call
// made 128-core hosts slower than 8-core ones).
class Pool {
 public:
  explicit Pool(unsigned n) : n_(n) {
    for (unsigned t = 0; t < n_; ++t) th_.emplace_back([this, t] { loop(t); });
  }
  ~Pool() {
    {
      std::lock_guard<std::mutex> l(m_);
      stop_ = true;
      ++gen_;
    }
    cv_.notify_all();
    for (auto& x : th_) x.join();
  }
  void run(const std::function<void(unsigned)>& f) {
    {
      std::lock_guard<std::mutex> l(m_);
      job_ = &f;
      left_ = n_;
      ++gen_;
    }
    cv_.notify_all();
    std::unique_lock<std::mutex> l(m_);
    done_.wait(l, [this] { return left_ == 0; });
  }
  unsigned size() const { return n_; }

 private:
  void loop(unsigned t) {
    uint64_t seen = 0;
    for (;;) {
      const std::function<void(unsigned)>* f;
      {
        std::unique_lock<std::mutex> l(m_);
        cv_.wait(l, [&] { return gen_ != seen; });
        seen = gen_;
        if (stop_) return;
        f = job_;
      }
      (*f)(t);
      {
        std::lock_guard<std::mutex> l(m_);
        if (--left_ == 0) done_.notify_all();
      }
    }
  }
  unsigned n_;
  std::vector<std::thread> th_;
  std::mutex m_;
  std::condition_variable cv_, done_;
  const std::function<void(unsigned)>* job_ = nullptr;
  unsigned left_ = 0;
  uint64_t gen_ = 0;
  bool stop_ = false;
};

struct jro_cluster {
  jr_config cfg;
  unsigned n_threads = 1;
  std::unique_ptr<Pool> pool;
  uint64_t step_index = 0;
  std::vector<Replica> reps;  // [g * R + (node-1)]
  std::vector<uint32_t> route;  // [g]: leader_id of the last jro_leader_table call (0 = none), for jro_run_tokens
  bool auto_trunc = false;      // jr_set_auto_truncate: every fused run ends with jro_truncate(auto_trunc_margin)
  uint32_t auto_trunc_margin = 0;
  Replica& at(uint32_t g, uint32_t node) { return reps[(size_t)g * cfg.n_replicas + (node - 1)]; }
};

namespace {

uint64_t synth_token(uint64_t step_index, uint32_t i, uint64_t g_global) {
  return ((step_index * 8 + i + 1) << 32) | (g_global & 0xffffffffull);
}

struct StepCtx {
  uint64_t now;
  uint32_t flags;
  uint32_t n_synth;
  const jr_proposal* proposals;
  // inject bucketed per replica: indices into args->inject
  const std::vector<std::vector<uint32_t>>* inject_idx;
  const jr_msg* inject;
  uint64_t step_index;
};

void step_group(jro_cluster* c, uint32_t g, const StepCtx& s) {
  const uint32_t R = c->cfg.n_replicas;
  const uint64_t gg = c->cfg.group_offset + g;
  for (uint32_t r = 1; r <= R; ++r) {
    Replica& me = c->at(g, r);
    Node& n = *me.node;
    // 1. peer mail of the previous step: ascending sender id, FIFO per sender
    if (s.flags & JR_STEP_DELIVER) {
      for (uint32_t sdr = 1; sdr <= R; ++sdr) {
        if (sdr == r) continue;
        for (const Message& m : c->at(g, sdr).prev_out) {
          bool mine = m.to.kind == JR_ADDR_PEERS || (m.to.kind == JR_ADDR_PEER && m.to.id == r);
          if (mine) n.apply(m.command, s.now);
        }
      }
    }
    // 2. host-injected commands
    if (s.inject_idx) {
      for (uint32_t idx : (*s.inject_idx)[(size_t)g * R + (r - 1)]) n.apply(from_abi(s.inject[idx]), s.now);
    }
    // 3. proposals
    if (s.proposals && s.proposals[g].node == r) {
      Command cr{JR_CMD_CLIENT_REQUEST};
      cr.req.id = s.proposals[g].token;
      cr.req.address = Address::client();
      n.apply(cr, s.now);
    }
    if (s.flags & JR_STEP_SYNTH_PROPOSALS) {
      for (uint32_t i = 0; i < s.n_synth; ++i) {
        if (n.role() != JR_ROLE_LEADER) break;
        Command cr{JR_CMD_CLIENT_REQUEST};
        cr.req.id = synth_token(s.step_index, i, gg);
        cr.req.address = Address::client();
        n.apply(cr, s.now);
      }
    }
    // 4. tick
    if (s.flags & JR_STEP_TICK) n.apply(Command{JR_CMD_TICK}, s.now);
  }
  // rotate mailboxes, fold digests
  const bool digests = (c->cfg.flags & JR_F_STREAM_DIGEST) != 0;
  const bool keep_fsm = (c->cfg.flags & JR_F_CAPTURE_FSM) != 0;
  for (uint32_t r = 1; r <= R; ++r) {
    Replica& me = c->at(g, r);
    Node& n = *me.node;
    if (digests) {
      for (const Message& m : n.rpc) {
        me.msg_digest = digest_msg(me.msg_digest, to_abi(m, g));
        ++me.n_msgs;
      }
      for (; me.fsm_digested < n.fsm.size(); ++me.fsm_digested) {
        me.fsm_digest = digest_fsm(me.fsm_digest, fsm_to_abi(n.fsm[me.fsm_digested], g, r));
        ++me.n_fsm;
      }
    }
    if (!keep_fsm) {  // fsm_tx with no receiver: drop
      n.fsm.clear();
      me.fsm_digested = 0;
    }
    me.prev_out.swap(n.rpc);
    n.rpc.clear();
  }
}

void for_groups(jro_cluster* c, const std::function<void(uint32_t, uint32_t)>& body) {
  const uint32_t G = c->cfg.n_groups;
  if (!c->pool) {
    body(0, G);
    return;
  }
  const unsigned T = c->pool->size();
  c->pool->run([&](unsigned t) { body((uint32_t)((uint64_t)G * t / T), (uint32_t)((uint64_t)G * (t + 1) / T)); });
}

void run_step(jro_cluster* c, const StepCtx& s) {
  for_groups(c, [&](uint32_t lo, uint32_t hi) {
    for (uint32_t g = lo; g < hi; ++g) step_group(c, g, s);
  });
  c->step_index++;
}

void clear_fsm(jro_cluster* c) {
  for (auto& r : c->reps) {
    r.node->fsm.clear();
    r.fsm_digested = 0;
  }
}

}  // namespace

extern "C" {

jr_status jro_create(const jr_config* cfg, unsigned n_threads, jro_cluster** out) {
  if (!cfg || !out) return JR_E_INVAL;
  if (cfg->abi_version != JR_ABI_VERSION) return JR_E_INVAL;
  if (cfg->n_replicas < 1 || cfg->n_replicas > JR_MAX_REPLICAS || cfg->n_groups < 1) return JR_E_INVAL;
  if (cfg->election_max_ms <= cfg->election_min_ms) return JR_E_INVAL;
  if (cfg->heartbeat_ms < 5 || cfg->election_min_ms < 5) return JR_E_INVAL;  // RaftConfig::validate, config.rs:70-75
  if (cfg->chain_capacity < 2) return JR_E_INVAL;
  auto* c = new jro_cluster();
  c->cfg = *cfg;
  c->n_threads = std::max(1u, std::min<unsigned>(n_threads ? n_threads : 1, cfg->n_groups));
  if (c->n_threads > 1) c->pool = std::make_unique<Pool>(c->n_threads);
  const uint32_t R = cfg->n_replicas;
  c->reps.resize((size_t)cfg->n_groups * R);
  c->route.assign(cfg->n_groups, 0u);
  // nodes are built by the worker that will step them (allocation locality)
  for_groups(c, [&](uint32_t glo, uint32_t ghi) {
  for (uint32_t g = glo; g < ghi; ++g) {
    for (uint32_t r = 1; r <= R; ++r) {
      NodeConfig nc;
      nc.id = r;
      for (uint32_t p = 1; p <= R; ++p)
        if (p != r) nc.peers.push_back(p);
      nc.seed = cfg->seed;
      nc.group = cfg->group_offset + g;
      nc.election_min_ms = cfg->election_min_ms;
      nc.election_max_ms = cfg->election_max_ms;
      nc.heartbeat_ms = cfg->heartbeat_ms;
      nc.chain_capacity = cfg->chain_capacity;
      nc.strict_commit_key = (cfg->flags & JR_F_SLED_COMMIT_KEY_STRICT) != 0;
      Replica& rep = c->at(g, r);
      rep.node = std::make_unique<Node>(nc);
      if (cfg->resident_mask && !((cfg->resident_mask >> (r - 1)) & 1u)) rep.node->alive = false;  // hosted elsewhere
      rep.msg_digest = rep.fsm_digest = mix64(((cfg->group_offset + g) << 8) | r);
    }
  }
  });
  *out = c;
  return JR_OK;
}

void jro_destroy(jro_cluster* c) { delete c; }

jr_status jro_step(jro_cluster* c, jr_step_args* a) {
  if (!c || !a) return JR_E_INVAL;
  const uint32_t R = c->cfg.n_replicas, G = c->cfg.n_groups;
  std::vector<std::vector<uint32_t>> idx;
  if (a->n_inject) {
    if (!a->inject) return JR_E_INVAL;
    idx.resize((size_t)G * R);
    for (size_t i = 0; i < a->n_inject; ++i) {
      const jr_msg& m = a->inject[i];
      if (m.group >= G || m.to_kind != JR_ADDR_PEER) return JR_E_INVAL;
      if (m.to_id < 1 || m.to_id > R) return JR_E_UNKNOWN_NODE;
      if (m.node_id > JR_MAX_NODE_ID || m.from_id > JR_MAX_NODE_ID || m.client_id > JR_MAX_NODE_ID) return JR_E_INVAL;
      if (m.kind == JR_CMD_VOTE_RESPONSE && (m.node_id < 1 || m.node_id > 32)) return JR_E_UNKNOWN_NODE;
      if (m.n_blocks > JR_MAX_AE_BLOCKS) return JR_E_INVAL;
      idx[(size_t)m.group * R + (m.to_id - 1)].push_back((uint32_t)i);
    }
  }
  if (a->proposals)
    for (uint32_t g = 0; g < G; ++g)
      if (a->proposals[g].node > R) return JR_E_UNKNOWN_NODE;
  clear_fsm(c);
  StepCtx s{a->now_ms, a->flags, a->n_synth, a->proposals, a->n_inject ? &idx : nullptr, a->inject, c->step_index};
  run_step(c, s);
  // capture
  size_t nm = 0, nf = 0;
  bool ovf = false;
  for (uint32_t g = 0; g < G; ++g)
    for (uint32_t r = 1; r <= R; ++r) {
      Replica& rep = c->at(g, r);
      if (c->cfg.flags & JR_F_CAPTURE_MESSAGES)
        for (const Message& m : rep.prev_out) {
          if (a->out_msgs && nm < a->cap_msgs) a->out_msgs[nm] = to_abi(m, g);
          else if (a->out_msgs) ovf = true;
          ++nm;
        }
      if (c->cfg.flags & JR_F_CAPTURE_FSM)
        for (const Instruction& i : rep.node->fsm) {
          if (a->out_fsm && nf < a->cap_fsm) a->out_fsm[nf] = fsm_to_abi(i, g, r);
          else if (a->out_fsm) ovf = true;
          ++nf;
        }
    }
  a->n_msgs = nm;
  a->n_fsm = nf;
  if (a->out_fsm) clear_fsm(c);  // returned to the caller: taken
  if (a->flags & JR_STEP_REPORT_FAULTS) {
    a->n_faulted = 0;
    for (auto& r : c->reps) a->n_faulted += r.node->fault() != 0;
  }
  return ovf ? JR_E_CAPACITY : JR_OK;
}

jr_status jro_truncate(jro_cluster* c, uint32_t margin);
// include/josefine_raft_abi.h jr_set_auto_truncate
jr_status jro_set_auto_truncate(jro_cluster* c, int enabled, uint32_t margin) {
  if (!c) return JR_E_INVAL;
  c->auto_trunc = enabled != 0;
  c->auto_trunc_margin = margin;
  return JR_OK;
}

jr_status jro_run(jro_cluster* c, uint64_t now0, uint32_t dt, uint32_t n_steps, uint32_t n_synth) {
  if (!c || n_synth > 8) return JR_E_INVAL;
  // Groups never interact, so each host thread runs ALL n_steps for its own
  // contiguous slice of groups: no barrier per step, no thread start per step.
  const uint64_t base = c->step_index;
  for_groups(c, [&](uint32_t lo, uint32_t hi) {
    for (uint32_t g = lo; g < hi; ++g)
      for (uint32_t k = 0; k < n_steps; ++k) {
        StepCtx s{now0 + (uint64_t)k * dt,
                  (uint32_t)(JR_STEP_DELIVER | JR_STEP_TICK | (n_synth ? JR_STEP_SYNTH_PROPOSALS : 0)),
                  n_synth, nullptr, nullptr, nullptr, base + k};
        step_group(c, g, s);
      }
  });
  c->step_index += n_steps;
  if (c->auto_trunc && n_steps) return jro_truncate(c, c->auto_trunc_margin);
  return JR_OK;
}

jr_status jro_run_proposals(jro_cluster* c, uint64_t now0, uint32_t dt, uint32_t n_steps, const jr_proposal* props,
                            uint32_t flags) {
  (void)flags;
  if (!c || !props) return JR_E_INVAL;
  const uint32_t G = c->cfg.n_groups;
  for (size_t i = 0; i < (size_t)n_steps * G; ++i)
    if (props[i].node > c->cfg.n_replicas) return JR_E_UNKNOWN_NODE;
  const uint64_t base = c->step_index;
  for_groups(c, [&](uint32_t lo, uint32_t hi) {
    for (uint32_t g = lo; g < hi; ++g)
      for (uint32_t k = 0; k < n_steps; ++k) {
        // step_group indexes proposals by group: point it at tick k's array
        StepCtx s{now0 + (uint64_t)k * dt, (uint32_t)(JR_STEP_DELIVER | JR_STEP_TICK), 0, props + (size_t)k * G,
                  nullptr, nullptr, base + k};
        step_group(c, g, s);
      }
  });
  c->step_index += n_steps;
  if (c->auto_trunc && n_steps) return jro_truncate(c, c->auto_trunc_margin);
  return JR_OK;
}

// include/josefine_raft_abi.h jr_run_tokens: tokens routed to the leader the last jro_leader_table call announced.
jr_status jro_run_tokens(jro_cluster* c, uint64_t now0, uint32_t dt, uint32_t n_steps, const uint64_t* tokens) {
  if (!c || !tokens) return JR_E_INVAL;
  const uint32_t G = c->cfg.n_groups;
  std::vector<jr_proposal> props((size_t)n_steps * G);
  for (size_t i = 0; i < props.size(); ++i) {
    props[i].token = tokens[i];
    props[i].node = tokens[i] ? c->route[i % G] : 0u;
    props[i].reserved = 0;
  }
  return jro_run_proposals(c, now0, dt, n_steps, props.data(), 0);
}

// include/josefine_raft_abi.h jr_run_token_runs: tokens[k*G + g] = base[g] + k * stride[g]
jr_status jro_run_token_runs(jro_cluster* c, uint64_t now0, uint32_t dt, uint32_t n_steps, const jr_token_run* runs) {
  if (!c || !runs) return JR_E_INVAL;
  const uint32_t G = c->cfg.n_groups;
  std::vector<uint64_t> tokens((size_t)n_steps * G);
  for (uint32_t k = 0; k < n_steps; ++k)
    for (uint32_t g = 0; g < G; ++g) tokens[(size_t)k * G + g] = runs[g].base ? runs[g].base + (uint64_t)k * runs[g].stride : 0;
  return jro_run_tokens(c, now0, dt, n_steps, tokens.data());
}

jr_status jro_drain_fsm(jro_cluster* c, jr_fsm_instr* out, size_t cap, size_t* n) {
  if (!c || !n) return JR_E_INVAL;
  size_t k = 0;
  bool ovf = false;
  if (c->cfg.flags & JR_F_CAPTURE_FSM)
    for (uint32_t g = 0; g < c->cfg.n_groups; ++g)
      for (uint32_t r = 1; r <= c->cfg.n_replicas; ++r)
        for (const Instruction& i : c->at(g, r).node->fsm) {
          if (out && k < cap) out[k] = fsm_to_abi(i, g, r);
          else if (out) ovf = true;
          ++k;
        }
  *n = k;
  clear_fsm(c);  // the drain takes them (ABI 2)
  return ovf ? JR_E_CAPACITY : JR_OK;
}

jr_status jro_query(jro_cluster* c, uint32_t group, uint32_t node, jr_replica_state* o) {
  if (!c || !o || group >= c->cfg.n_groups || node < 1 || node > c->cfg.n_replicas) return JR_E_INVAL;
  const Node& n = *c->at(group, node).node;
  std::memset(o, 0, sizeof *o);
  o->current_term = n.current_term;
  o->voted_for = n.voted_for.value_or(0);
  o->leader_id = n.leader_id.value_or(0);
  o->election_time_ms = n.election_time;
  o->election_timeout_ms = n.election_timeout;
  o->rng_draws = n.rng_draws;
  o->head = n.chain.get_head();
  o->commit = n.chain.get_commit();
  o->id_gen = n.chain.id_gen();
  o->max_key = n.chain.blocks().empty() ? 0 : n.chain.blocks().rbegin()->first;
  if (n.role() == JR_ROLE_LEADER) {
    o->heartbeat_time_ms = n.heartbeat_time;
    for (auto& kv : n.progress->all()) {
      o->progress_head[kv.first - 1] = kv.second.head;
      if (kv.second.kind == NodeProgress::Replicate) o->progress_replicate |= 1u << (kv.first - 1);
    }
  }
  if (n.role() == JR_ROLE_CANDIDATE) {
    for (auto& kv : n.election->votes()) {
      o->votes_seen |= 1u << (kv.first - 1);
      if (kv.second) o->votes_granted |= 1u << (kv.first - 1);
    }
  }
  o->role = (uint8_t)n.role();
  o->fault = (uint8_t)n.fault();
  o->alive = n.alive;
  o->n_queued = (uint8_t)n.queued_reqs.size();
  o->chain_floor = n.chain.floor();
  return JR_OK;
}

jr_status jro_chain_read(jro_cluster* c, uint32_t group, uint32_t node, uint64_t first, uint32_t n,
                         jr_block* out, uint8_t* present) {
  if (!c || group >= c->cfg.n_groups || node < 1 || node > c->cfg.n_replicas) return JR_E_INVAL;
  const auto& db = c->at(group, node).node->chain.blocks();
  for (uint32_t i = 0; i < n; ++i) {
    auto it = db.find(first + i);
    if (present) present[i] = it != db.end();
    if (out) out[i] = it != db.end() ? jr_block{it->second.id, it->second.next, it->second.data} : jr_block{first + i, 0, 0};
  }
  return JR_OK;
}

// Normative state digest (DESIGN.md "Digests").
jr_status jro_state_digest(jro_cluster* c, uint64_t* out) {
  if (!c || !out) return JR_E_INVAL;
  uint64_t total = 0;
  const uint32_t R = c->cfg.n_replicas;
  for (uint32_t g = 0; g < c->cfg.n_groups; ++g)
    for (uint32_t r = 1; r <= R; ++r) {
      const Node& n = *c->at(g, r).node;
      uint64_t h = mix64(0x243f6a8885a308d3ull ^ (((c->cfg.group_offset + g) << 8) | r));
      h = fold(h, n.current_term);
      h = fold(h, n.voted_for.value_or(0));
      h = fold(h, (uint64_t)n.role() | ((uint64_t)n.fault() << 8) | ((uint64_t)(n.alive ? 1 : 0) << 16) |
                      ((uint64_t)n.queued_reqs.size() << 24));
      h = fold(h, n.election_time);
      h = fold(h, (uint64_t)n.election_timeout | ((uint64_t)n.rng_draws << 32));
      h = fold(h, n.chain.get_head());
      h = fold(h, n.chain.get_commit());
      h = fold(h, n.chain.id_gen());
      if (n.role() == JR_ROLE_FOLLOWER) h = fold(h, n.leader_id.value_or(0));
      if (n.role() == JR_ROLE_CANDIDATE) {
        uint64_t seen = 0, granted = 0;
        for (auto& kv : n.election->votes()) {
          seen |= 1ull << (kv.first - 1);
          if (kv.second) granted |= 1ull << (kv.first - 1);
        }
        h = fold(h, seen | (granted << 32));
      }
      if (n.role() == JR_ROLE_LEADER) {
        h = fold(h, n.heartbeat_time);
        uint64_t mask = 0;
        for (uint32_t i = 1; i <= R; ++i) {
          const NodeProgress& p = n.progress->all().at(i);
          h = fold(h, p.head);
          if (p.kind == NodeProgress::Replicate) mask |= 1ull << (i - 1);
        }
        h = fold(h, mask);
      }
      for (auto& q : n.queued_reqs) {
        h = fold(h, q.id);
        h = fold(h, (uint64_t)q.address.kind | ((uint64_t)q.address.id << 8));
      }
      uint64_t chain = 0;
      for (auto& kv : n.chain.blocks())
        chain += mix64(mix64(kv.second.id + 0x13198a2e03707344ull) ^ (kv.second.next * 0xa4093822299f31d1ull) ^ kv.second.data);
      h = fold(h, chain);
      total += h;
    }
  *out = total;
  return JR_OK;
}

jr_status jro_stream_digest(jro_cluster* c, uint64_t* md, uint64_t* fd, uint64_t* nm, uint64_t* nf) {
  if (!c) return JR_E_INVAL;
  if (!(c->cfg.flags & JR_F_STREAM_DIGEST)) return JR_E_INVAL;
  uint64_t a = 0, b = 0, x = 0, y = 0;
  for (auto& r : c->reps) {
    a += r.msg_digest;
    b += r.fsm_digest;
    x += r.n_msgs;
    y += r.n_fsm;
  }
  if (md) *md = a;
  if (fd) *fd = b;
  if (nm) *nm = x;
  if (nf) *nf = y;
  return JR_OK;
}

jr_status jro_fault_count(jro_cluster* c, uint64_t* n) {
  if (!c || !n) return JR_E_INVAL;
  uint64_t k = 0;
  for (auto& r : c->reps) k += r.node->fault() != 0;
  *n = k;
  return JR_OK;
}

jr_status jro_compact(jro_cluster* c) {
  if (!c) return JR_E_INVAL;
  for (auto& r : c->reps)
    if (r.node->alive && r.node->fault() == 0) r.node->chain.compact();
  return JR_OK;
}

// include/josefine_raft_abi.h jr_truncate (deviation D7)
jr_status jro_truncate(jro_cluster* c, uint32_t margin) {
  if (!c) return JR_E_INVAL;
  for (uint32_t g = 0; g < c->cfg.n_groups; ++g) {
    uint64_t lo = UINT64_MAX;
    for (uint32_t r = 1; r <= c->cfg.n_replicas; ++r) {
      const Node& n = *c->at(g, r).node;
      if (n.alive && n.fault() == 0) lo = std::min<uint64_t>(lo, n.chain.get_commit());
    }
    if (lo == UINT64_MAX) continue;
    const uint64_t floor = lo > margin ? lo - margin : 0;
    for (uint32_t r = 1; r <= c->cfg.n_replicas; ++r) c->at(g, r).node->chain.truncate(floor);
  }
  return JR_OK;
}

// include/josefine_raft_abi.h jr_node_restart: RaftHandle::new over an existing data directory
jr_status jro_node_restart(jro_cluster* c, uint32_t group, uint32_t node, uint64_t now_ms, const jr_block* blocks,
                           size_t n_blocks, uint64_t commit, int commit_key) {
  if (!c || group >= c->cfg.n_groups || node < 1 || node > c->cfg.n_replicas || (n_blocks && !blocks)) return JR_E_INVAL;
  Replica& rep = c->at(group, node);
  const uint64_t floor = rep.node->chain.floor();
  if (commit >= JR_BLOCK_ID_LIMIT) return JR_E_INVAL;  // D4
  std::vector<Block> persisted;
  for (size_t k = 0; k < n_blocks; ++k) {
    if (blocks[k].id < floor || blocks[k].id - floor >= c->cfg.chain_capacity) return JR_E_INVAL;
    if (blocks[k].id >= JR_BLOCK_ID_LIMIT || blocks[k].next >= JR_BLOCK_ID_LIMIT) return JR_E_INVAL;  // D4
    persisted.push_back(Block{blocks[k].id, blocks[k].next, blocks[k].data});
  }
  NodeConfig nc = rep.node->config();
  const bool strict = (c->cfg.flags & JR_F_SLED_COMMIT_KEY_STRICT) != 0;
  std::vector<Instruction> undrained = std::move(rep.node->fsm);   // what the old incarnation emitted is still owed to the host
  rep.node = std::make_unique<Node>(nc, Chain(c->cfg.chain_capacity, strict, persisted, commit, commit_key != 0, floor), now_ms);
  rep.node->fsm = std::move(undrained);
  rep.prev_out.clear();
  return JR_OK;
}

// Test-only: moves every group's block ids up by k with f(v) = v + k for v >= F, v for v < F, F = the group's floor.
// f keeps every order, equality and the literal 0 (F > 0), and commutes with what Raft does with ids, so the shifted
// cluster's future is the old one's future shifted by f -- until an id reaches 2^31 (D4).  Only between steps with no
// mail and no undrained Instruction (they carry ids too), every floor above 0 and every shifted id below 2^31;
// JR_E_INVAL otherwise, with nothing changed.
jr_status jro_shift_ids(jro_cluster* c, uint64_t k) {
  if (!c) return JR_E_INVAL;
  const uint32_t R = c->cfg.n_replicas;
  for (uint32_t g = 0; g < c->cfg.n_groups; ++g) {
    const uint64_t floor = c->at(g, 1).node->chain.floor();
    if (floor == 0 || k >= JR_BLOCK_ID_LIMIT) return JR_E_INVAL;
    auto bad = [&](uint64_t v) { return v >= floor && v + k >= JR_BLOCK_ID_LIMIT; };
    for (uint32_t r = 1; r <= R; ++r) {
      const Replica& rep = c->at(g, r);
      const Node& n = *rep.node;
      const Chain& ch = n.chain;
      if (!rep.prev_out.empty() || !n.rpc.empty() || !n.fsm.empty() || ch.floor() != floor) return JR_E_INVAL;
      if (bad(floor) || bad(ch.get_head()) || bad(ch.get_commit()) || bad(ch.id_gen())) return JR_E_INVAL;
      for (auto& kv : ch.blocks())
        if (bad(kv.first) || bad(kv.second.next)) return JR_E_INVAL;
      if (n.progress)
        for (auto& kv : n.progress->all())
          if (bad(kv.second.head)) return JR_E_INVAL;
    }
  }
  for (uint32_t g = 0; g < c->cfg.n_groups; ++g)
    for (uint32_t r = 1; r <= R; ++r) {
      Node& n = *c->at(g, r).node;
      const uint64_t floor = n.chain.floor();
      n.chain.shift_ids(k);
      if (n.progress)
        for (auto& kv : n.progress->all_mut())
          if (kv.second.head >= floor) kv.second.head += k;
    }
  return JR_OK;
}

jr_status jro_set_alive(jro_cluster* c, uint32_t group, uint32_t node, int alive) {
  if (!c || group >= c->cfg.n_groups || node < 1 || node > c->cfg.n_replicas) return JR_E_INVAL;
  c->at(group, node).node->alive = alive != 0;
  return JR_OK;
}

jr_status jro_kill_leaders(jro_cluster* c, uint64_t salt, uint32_t permille, uint64_t* n_killed) {
  if (!c) return JR_E_INVAL;
  uint64_t k = 0;
  uint64_t base = mix64(c->cfg.seed ^ salt);
  for (uint32_t g = 0; g < c->cfg.n_groups; ++g) {
    if (mix64(base + c->cfg.group_offset + g) % 1000 >= permille) continue;
    for (uint32_t r = 1; r <= c->cfg.n_replicas; ++r) {
      Node& n = *c->at(g, r).node;
      if (n.alive && n.fault() == 0 && n.role() == JR_ROLE_LEADER) {
        n.alive = false;
        ++k;
      }
    }
  }
  if (n_killed) *n_killed = k;
  return JR_OK;
}

jr_status jro_leader_table(jro_cluster* c, jr_leader_entry* out) {
  if (!c || !out) return JR_E_INVAL;
  for (uint32_t g = 0; g < c->cfg.n_groups; ++g) {
    jr_leader_entry e{0, 0, 0};
    for (uint32_t r = 1; r <= c->cfg.n_replicas; ++r) {
      const Node& n = *c->at(g, r).node;
      if (!n.alive || n.fault() != 0 || n.role() != JR_ROLE_LEADER) continue;
      if (e.leader_id == 0 || n.current_term >= e.term) {  // ties: higher id wins (ascending scan)
        e.term = n.current_term;
        e.leader_id = r;
        e.commit = (uint32_t)n.chain.get_commit();
      }
    }
    out[g] = e;
    c->route[g] = e.leader_id;
  }
  return JR_OK;
}

uint32_t jro_election_timeout(uint64_t seed, uint64_t group, uint32_t node, uint32_t draw, uint32_t mn, uint32_t mx) {
  return election_timeout_draw(seed, group, node, draw, mn, mx);
}

// ---- direct Chain access for the ported chain.rs known-answer tests -------------
struct jro_chain {
  Chain chain;
  int fault = 0;
};
jro_chain* jro_chain_new(uint64_t capacity, int strict) { return new jro_chain{Chain(capacity, strict != 0), 0}; }
void jro_chain_free(jro_chain* c) { delete c; }
int jro_chain_fault(jro_chain* c) { return c->fault; }
#define CHAIN_TRY(stmt) \
  try { stmt; } catch (const Fault& f) { c->fault = f.code; }
uint64_t jro_chain_append(jro_chain* c, uint64_t data) {
  uint64_t id = 0;
  CHAIN_TRY(id = c->chain.append(data));
  return id;
}
void jro_chain_extend(jro_chain* c, uint64_t id, uint64_t next, uint64_t data) { CHAIN_TRY(c->chain.extend(Block{id, next, data})); }
void jro_chain_commit(jro_chain* c, uint64_t id) { CHAIN_TRY(c->chain.commit(id)); }
int jro_chain_has(jro_chain* c, uint64_t id) { return c->chain.has(id); }
void jro_chain_compact(jro_chain* c) { c->chain.compact(); }
uint64_t jro_chain_head(jro_chain* c) { return c->chain.get_head(); }
uint64_t jro_chain_commit_id(jro_chain* c) { return c->chain.get_commit(); }
size_t jro_chain_len(jro_chain* c) { return c->chain.blocks().size(); }
// range(lo..) skip/take; returns count, fills ids
size_t jro_chain_range_from(jro_chain* c, uint64_t lo, size_t skip, size_t take, uint64_t* ids, size_t cap) {
  size_t k = 0;
  CHAIN_TRY(for (auto& b : c->chain.range_from_skip_take(lo, skip, take)) { if (k < cap) ids[k] = b.id; ++k; });
  return k;
}

}  // extern "C"
