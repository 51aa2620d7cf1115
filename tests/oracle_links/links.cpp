// TEST INFRASTRUCTURE ONLY: the oracle's restatement of the peer-link calls (include/josefine_raft_abi.h, "peer
// links", deviation D8).  Built into its own library together with the unchanged oracle sources: this translation unit
// includes restated_cluster.cpp, so the cluster's Replica objects are visible here.
//
// The matrices live in a table beside the cluster (the oracle's struct is not ours to extend).  Delivery takes them into
// account through jrl_route_mail, which a host calls in front of every single step: it rewrites each sender's mail of
// the previous step into the mail a network with these cuts delivers -- a Peer(r) message over a cut link is removed,
// and a Peers broadcast becomes, in its place, one Peer(r) copy per receiver r whose link from the sender is up.  Every
// receiver then finds exactly its deliverable mail, in the same order, and step_group applies it unchanged.  The next
// step replaces the rewritten mail with the new emission, and the stream digests were folded at emission, so nothing
// else ever sees the rewrite.
#include "restated_cluster.cpp"

#include <map>

namespace {
std::mutex g_mu;
std::map<const jro_cluster*, std::vector<uint64_t>> g_links;   // [cluster][group]; absent = fully connected

std::vector<uint64_t>& links_of(const jro_cluster* c) {
  auto& v = g_links[c];
  if (v.size() != c->cfg.n_groups) v.assign(c->cfg.n_groups, 0);
  return v;
}

uint64_t valid_mask(uint32_t R) {
  uint64_t m = 0;
  for (uint32_t r = 0; r < R; ++r) m |= (((1ull << R) - 1ull) & ~(1ull << r)) << (8u * r);
  return m;
}

bool check_groups(const jro_cluster* c, const uint32_t* groups, size_t n) {
  if (!(c->cfg.flags & JR_F_PEER_LINKS)) return false;
  if (!groups) return n == c->cfg.n_groups;
  std::vector<uint8_t> seen(c->cfg.n_groups, 0);
  for (size_t k = 0; k < n; ++k) {
    if (groups[k] >= c->cfg.n_groups || seen[groups[k]]) return false;
    seen[groups[k]] = 1;
  }
  return true;
}
}  // namespace

extern "C" {

jr_status jro_set_links(jro_cluster* c, const uint32_t* groups, const uint64_t* cuts, size_t n) {
  if (!c || (n && !cuts) || !check_groups(c, groups, n)) return JR_E_INVAL;
  const uint64_t bad = ~valid_mask(c->cfg.n_replicas);
  for (size_t k = 0; k < n; ++k)
    if (cuts[k] & bad) return JR_E_INVAL;
  std::lock_guard<std::mutex> l(g_mu);
  auto& v = links_of(c);
  for (size_t k = 0; k < n; ++k) v[groups ? groups[k] : k] = cuts[k];
  return JR_OK;
}

jr_status jro_get_links(jro_cluster* c, const uint32_t* groups, size_t n, uint64_t* out) {
  if (!c || (n && !out) || !check_groups(c, groups, n)) return JR_E_INVAL;
  std::lock_guard<std::mutex> l(g_mu);
  auto& v = links_of(c);
  for (size_t k = 0; k < n; ++k) out[k] = v[groups ? groups[k] : k];
  return JR_OK;
}

// jro_kill_leaders' selection; every link to and from each live leader of a picked group is cut.
jr_status jro_isolate_leaders(jro_cluster* c, uint64_t salt, uint32_t permille, uint64_t* n_isolated) {
  if (!c || !(c->cfg.flags & JR_F_PEER_LINKS)) return JR_E_INVAL;
  const uint32_t R = c->cfg.n_replicas;
  std::lock_guard<std::mutex> l(g_mu);
  auto& v = links_of(c);
  uint64_t k = 0;
  const uint64_t base = mix64(c->cfg.seed ^ salt);
  for (uint32_t g = 0; g < c->cfg.n_groups; ++g) {
    if (mix64(base + c->cfg.group_offset + g) % 1000 >= permille) continue;
    uint64_t m = 0;
    bool had = false;   // a live leader (at R = 1 it has no link to cut, and still counts)
    for (uint32_t r = 1; r <= R; ++r) {
      const Node& n = *c->at(g, r).node;
      if (!(n.alive && n.fault() == 0 && n.role() == JR_ROLE_LEADER)) continue;
      had = true;
      for (uint32_t q = 1; q <= R; ++q)
        if (q != r) m |= (1ull << (8 * (r - 1) + (q - 1))) | (1ull << (8 * (q - 1) + (r - 1)));
    }
    if (had) ++k;
    v[g] |= m;
  }
  if (n_isolated) *n_isolated = k;
  return JR_OK;
}

// The mail of the previous step, as the cut network delivers it (see the top of this file).  Only groups with a cut.
jr_status jrl_route_mail(jro_cluster* c) {
  if (!c) return JR_E_INVAL;
  std::lock_guard<std::mutex> l(g_mu);
  auto it = g_links.find(c);
  if (it == g_links.end()) return JR_OK;
  const uint32_t R = c->cfg.n_replicas;
  for (uint32_t g = 0; g < c->cfg.n_groups; ++g) {
    const uint64_t cut = it->second[g];
    if (!cut) continue;
    for (uint32_t s = 1; s <= R; ++s) {
      std::vector<Message>& out = c->at(g, s).prev_out;
      std::vector<Message> routed;
      for (const Message& m : out) {
        const bool peers = m.to.kind == JR_ADDR_PEERS;
        if (!peers && m.to.kind != JR_ADDR_PEER) continue;   // not peer mail: no receiver takes it
        for (uint32_t r = 1; r <= R; ++r) {
          if (r == s || (!peers && m.to.id != r) || ((cut >> (8 * (r - 1) + (s - 1))) & 1u)) continue;
          routed.push_back(m);
          routed.back().to = Address{JR_ADDR_PEER, r};
        }
      }
      out.swap(routed);
    }
  }
  return JR_OK;
}

// jro_destroy, and the cluster's matrices with it (a later cluster may get the same address).
void jrl_destroy(jro_cluster* c) {
  {
    std::lock_guard<std::mutex> l(g_mu);
    g_links.erase(c);
  }
  jro_destroy(c);
}

}  // extern "C"
