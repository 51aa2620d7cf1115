// TEST INFRASTRUCTURE ONLY: jro_group_move, the oracle's restatement of jr_group_export + jr_group_import
// (include/josefine_raft_abi.h, "moving groups between engines").  Built into its own library together with the
// unchanged oracle sources: this translation unit includes restated_cluster.cpp, so the cluster's Replica objects and
// route table are visible here.
#include "restated_cluster.cpp"

namespace {
// A moved node draws its election timeouts under the destination's D2 key, which lives in the node's private config.
// Explicit instantiation is exempt from access checks: Rob hands out a pointer to that member without touching the
// oracle's class.
struct NodeCfg {
  using type = restated::NodeConfig restated::Node::*;
  friend type node_cfg(NodeCfg);
};
template <typename Tag, typename Tag::type M>
struct Rob {
  friend typename Tag::type node_cfg(Tag) { return M; }
};
template struct Rob<NodeCfg, &restated::Node::cfg_>;

void rekey(restated::Node& n, uint64_t seed, uint64_t group) {
  restated::NodeConfig& c = n.*node_cfg(NodeCfg{});
  c.seed = seed;
  c.group = group;
}
}  // namespace

extern "C" {

// Group groups[j] of src becomes slot slots[j] of dst, with every replica, its mail in flight, its undrained
// Instructions and its route entry; each node takes dst's D2 key.  The source replicas stay behind silenced, with empty
// Instruction buffers.  src == dst moves groups between slots of one cluster.  JR_E_INVAL, nothing moved, for the
// configurations and lists jr_group_import refuses.
jr_status jro_group_move(jro_cluster* src, jro_cluster* dst, const uint32_t* groups, const uint32_t* slots, size_t n) {
  if (!src || !dst || (n && (!groups || !slots))) return JR_E_INVAL;
  const jr_config &a = src->cfg, &b = dst->cfg;
  const uint32_t keep = ~(uint32_t)JR_F_NO_SYMMETRIC_FOLD;
  if (a.n_replicas != b.n_replicas || a.chain_capacity != b.chain_capacity || a.mailbox_units != b.mailbox_units ||
      a.fsm_units != b.fsm_units || a.election_min_ms != b.election_min_ms || a.election_max_ms != b.election_max_ms ||
      a.heartbeat_ms != b.heartbeat_ms || a.resident_mask != b.resident_mask || (a.flags & keep) != (b.flags & keep))
    return JR_E_INVAL;
  std::vector<uint8_t> seen_g(a.n_groups, 0), seen_s(b.n_groups, 0);
  for (size_t j = 0; j < n; ++j) {
    if (groups[j] >= a.n_groups || seen_g[groups[j]] || slots[j] >= b.n_groups || seen_s[slots[j]]) return JR_E_INVAL;
    seen_g[groups[j]] = seen_s[slots[j]] = 1;
  }
  const uint32_t R = a.n_replicas;
  std::vector<Replica> moved(n * R);
  std::vector<uint32_t> route(n);
  for (size_t j = 0; j < n; ++j) {   // copies first: src and dst may be the same cluster
    for (uint32_t r = 1; r <= R; ++r) {
      const Replica& s = src->at(groups[j], r);
      Replica& m = moved[j * R + (r - 1)];
      m.node = std::make_unique<restated::Node>(*s.node);
      m.prev_out = s.prev_out;
      m.msg_digest = s.msg_digest;
      m.fsm_digest = s.fsm_digest;
      m.n_msgs = s.n_msgs;
      m.n_fsm = s.n_fsm;
      m.fsm_digested = s.fsm_digested;
    }
    route[j] = src->route[groups[j]];
  }
  for (size_t j = 0; j < n; ++j)   // detach
    for (uint32_t r = 1; r <= R; ++r) {
      Replica& s = src->at(groups[j], r);
      s.node->alive = false;
      s.node->fsm.clear();
      s.fsm_digested = 0;
    }
  for (size_t j = 0; j < n; ++j) {
    for (uint32_t r = 1; r <= R; ++r) {
      Replica& d = dst->at(slots[j], r);
      d = std::move(moved[j * R + (r - 1)]);
      rekey(*d.node, b.seed, b.group_offset + slots[j]);
    }
    dst->route[slots[j]] = route[j];
  }
  return JR_OK;
}

}  // extern "C"
