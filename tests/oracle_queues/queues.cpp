// TEST INFRASTRUCTURE ONLY: the oracle's restatement of the link queues (include/josefine_raft_abi.h, "link queues",
// deviation D8).  One translation unit with the peer-link restatement (links.cpp, which includes restated_cluster.cpp),
// so the cluster's Replica objects and the link matrices are visible here.
//
// Each (group, sender s, receiver r) has a FIFO of oracle Messages beside the cluster.  jrq_route_mail, called in front of
// every single step, rewrites each sender's mail of the previous step into what the network with these cuts and queues
// delivers, as jrl_route_mail does for plain cuts:
//   * a step that delivers nothing (no JR_STEP_DELIVER) changes nothing: its mail is dropped as all undelivered mail is;
//   * a Message for r over a cut link s -> r goes to the back of that link's queue while it holds fewer than
//     JR_LINK_QUEUE_MSGS Messages, and is dropped otherwise (each oracle Message is one Message);
//   * a link s -> r that is up with a non-empty queue: the queue, as Peer(r) copies, goes in front of s's routed mail,
//     and the queue is emptied;
//   * a Peers broadcast becomes one Peer(r) copy per receiver r whose link from s is up.
// Groups with a zero matrix are visited too while they have queued mail.  An engine without JR_F_LINK_QUEUES gets
// jrl_route_mail unchanged.
#include "links.cpp"

#include <deque>

namespace {
std::map<const jro_cluster*, std::vector<std::deque<Message>>> g_queues;   // [cluster][(g * R + (r-1)) * R + (s-1)]

std::vector<std::deque<Message>>& queues_of(const jro_cluster* c) {
  auto& v = g_queues[c];
  const size_t R = c->cfg.n_replicas;
  if (v.size() != c->cfg.n_groups * R * R) v.assign(c->cfg.n_groups * R * R, {});
  return v;
}

bool queues_on(const jro_cluster* c) { return (c->cfg.flags & JR_F_LINK_QUEUES) != 0; }
}  // namespace

extern "C" {

jr_status jrq_route_mail(jro_cluster* c, int deliver) {
  if (!c) return JR_E_INVAL;
  if (!queues_on(c)) return jrl_route_mail(c);
  if (!deliver) return JR_OK;
  std::lock_guard<std::mutex> l(g_mu);
  auto& Q = queues_of(c);
  auto it = g_links.find(c);
  const uint32_t R = c->cfg.n_replicas;
  for (uint32_t g = 0; g < c->cfg.n_groups; ++g) {
    const uint64_t cut = it == g_links.end() ? 0 : it->second[g];
    bool queued = false;
    for (size_t k = (size_t)g * R * R; k < (size_t)(g + 1) * R * R && !queued; ++k) queued = !Q[k].empty();
    if (!cut && !queued) continue;
    for (uint32_t s = 1; s <= R; ++s) {
      std::vector<Message>& out = c->at(g, s).prev_out;
      std::vector<Message> routed;
      for (uint32_t r = 1; r <= R; ++r) {   // replay: the queues of the links from s that are up
        std::deque<Message>& q = Q[((size_t)g * R + (r - 1)) * R + (s - 1)];
        if (r == s || ((cut >> (8 * (r - 1) + (s - 1))) & 1u) || q.empty()) continue;
        for (const Message& m : q) {
          routed.push_back(m);
          routed.back().to = Address{JR_ADDR_PEER, r};
        }
        q.clear();
      }
      for (const Message& m : out) {
        const bool peers = m.to.kind == JR_ADDR_PEERS;
        if (!peers && m.to.kind != JR_ADDR_PEER) continue;   // not peer mail: no receiver takes it
        for (uint32_t r = 1; r <= R; ++r) {
          if (r == s || (!peers && m.to.id != r)) continue;
          Message copy = m;
          copy.to = Address{JR_ADDR_PEER, r};
          if ((cut >> (8 * (r - 1) + (s - 1))) & 1u) {
            std::deque<Message>& q = Q[((size_t)g * R + (r - 1)) * R + (s - 1)];
            if (q.size() < JR_LINK_QUEUE_MSGS) q.push_back(copy);
          } else {
            routed.push_back(copy);
          }
        }
      }
      out.swap(routed);
    }
  }
  return JR_OK;
}

// jr_get_link_queues: depths[64*i + 8*(r-1) + (s-1)].
jr_status jro_get_link_queues(jro_cluster* c, const uint32_t* groups, size_t n, uint8_t* depths) {
  if (!c || (n && !depths) || !queues_on(c) || !check_groups(c, groups, n)) return JR_E_INVAL;
  std::lock_guard<std::mutex> l(g_mu);
  auto& Q = queues_of(c);
  const uint32_t R = c->cfg.n_replicas;
  memset(depths, 0, 64 * n);
  for (size_t k = 0; k < n; ++k) {
    const uint32_t g = groups ? groups[k] : (uint32_t)k;
    for (uint32_t r = 1; r <= R; ++r)
      for (uint32_t s = 1; s <= R; ++s)
        depths[64 * k + 8 * (r - 1) + (s - 1)] = (uint8_t)Q[((size_t)g * R + (r - 1)) * R + (s - 1)].size();
  }
  return JR_OK;
}

// The queues FROM node `node` of `group` are gone (jr_node_restart: a new process has new channels).
jr_status jrq_drop_sender(jro_cluster* c, uint32_t group, uint32_t node) {
  if (!c || group >= c->cfg.n_groups || node < 1 || node > c->cfg.n_replicas) return JR_E_INVAL;
  std::lock_guard<std::mutex> l(g_mu);
  auto& Q = queues_of(c);
  const uint32_t R = c->cfg.n_replicas;
  for (uint32_t r = 1; r <= R; ++r) Q[((size_t)group * R + (r - 1)) * R + (node - 1)].clear();
  return JR_OK;
}

// jr_engine_reset's share: every queue empty.
jr_status jrq_reset(jro_cluster* c) {
  if (!c) return JR_E_INVAL;
  std::lock_guard<std::mutex> l(g_mu);
  for (auto& q : queues_of(c)) q.clear();
  return JR_OK;
}

void jrq_destroy(jro_cluster* c) {
  {
    std::lock_guard<std::mutex> l(g_mu);
    g_queues.erase(c);
  }
  jrl_destroy(c);
}

}  // extern "C"
