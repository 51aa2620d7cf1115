// engine.cu -- kernels + C ABI of the H100 batched Chained-Raft engine.
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a (see __graft_entry__.build).
// No CPU fallback: without a CUDA device jr_engine_create returns JR_E_NO_DEVICE.
//
// Reference interfaces replaced are cited in include/josefine_raft_abi.h; the
// replica state machine is in raft_device.cuh.
#include <algorithm>
#include <atomic>
#include <cassert>
#include <chrono>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <condition_variable>
#include <mutex>
#include <new>
#include <thread>
#include <vector>

#include "raft_device.cuh"
#include "sym_fold.cuh"

using namespace jr;

// ============================================================================
// kernels
// ============================================================================

// n_ticks fused schedule steps for every replica.  CTA = 32 groups x R warps; warp w
// is replica w of those groups.  Replica state lives in registers for the whole
// launch; the mailboxes of the CTA's groups live in shared memory (double
// buffered, units beyond Us spill to the global mailbox); block-table reads go
// through a per-lane shared-memory cache.  Groups never interact, so the only
// synchronisation between ticks is __syncthreads().
// A split launch (p0.n_parts > 1) runs every block's ticks as n_parts consecutive tasks.  Tasks are taken by
// ticket, in launch order, so all part k-1 tasks are running or done before any part k task starts; a part k
// task waits for its block's part k-1 (release/acquire on d.done[block]) and then continues from the state
// and mailboxes that task stored -- exactly what the next launch would do.  The point is the last wave:
// 600 equal tasks on 528 CTA slots (132 SMs x 4) take 2 rounds, 1200 half-length tasks take 3 half-rounds.
#ifdef JR_EMU
#ifdef JR_EMU_BREAK_HANDOFF  // negative control of tests/emu/tsan_split.cpp: the race detector must notice this
#define JR_EMU_HANDOFF_ACQUIRE __ATOMIC_RELAXED
#define JR_EMU_HANDOFF_RELEASE __ATOMIC_RELAXED
#else
#define JR_EMU_HANDOFF_ACQUIRE __ATOMIC_ACQUIRE
#define JR_EMU_HANDOFF_RELEASE __ATOMIC_RELEASE
#endif
#endif
__device__ __forceinline__ uint32_t ld_acquire_u32(const uint32_t* p) {
#ifdef JR_EMU
  return __atomic_load_n(p, JR_EMU_HANDOFF_ACQUIRE);
#else
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
#endif
}
__device__ __forceinline__ void st_release_u32(uint32_t* p, uint32_t v) {
#ifdef JR_EMU
  __atomic_store_n(p, v, JR_EMU_HANDOFF_RELEASE);
#else
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
#endif
}

// Resident CTAs the register allocation must allow (the kernel is latency bound: occupancy is throughput).
// R = 5 (160 threads) holds 4 CTAs per SM at 96 registers, what ptxas picked on its own before the stream encoder
// was added; the other sizes keep their natural allocation.
constexpr int step_min_ctas(int R) { return (R == 4 || R == 5) ? 4 : 1; }

// QUEUES: the engine has JR_F_LINK_QUEUES (cut mail is queued and replayed, raft_device.cuh); a separate instantiation,
// so the other engines' kernel keeps its code and registers.
template <int R, bool SORTED, bool QUEUES = false>
__global__ void __launch_bounds__(32 * R, step_min_ctas(R)) step_kernel(const Dev d, const StepParams p0) {
  JR_DYN_SMEM(uint4, smem);
  const uint32_t w = threadIdx.x >> 5, lane = threadIdx.x & 31u;
  StepParams p = p0;
  uint32_t blk = blockIdx.x, part = 0;
  if (p0.n_parts > 1) {
    uint32_t* s_ticket = reinterpret_cast<uint32_t*>(smem);  // free until stage_inbox: fenced by the two barriers
    if (threadIdx.x == 0) *s_ticket = atomicAdd(d.scatter + 1, 1u) - p0.ticket_base;
    __syncthreads();
    const uint32_t ticket = *s_ticket;
    __syncthreads();
    part = ticket / p0.n_blocks;
    blk = ticket - part * p0.n_blocks;
    const uint32_t t0 = part * p0.part_ticks;  // host: (n_parts - 1) * part_ticks < n_ticks
    p.n_ticks = min(p0.part_ticks, p0.n_ticks - t0);
    p.now += (uint64_t)t0 * p0.dt;
    p.step_index += t0;
    p.cur ^= (int)(t0 & 1u);
    if (p.proposals) p.proposals += (size_t)t0 * p0.prop_stride;
    p.tok_tick += t0;
    if (part) {
      p.phases = PH_RESET_OUT | PH_DRAIN | PH_PROPOSE | PH_TICK;
      if (threadIdx.x == 0)
        while (ld_acquire_u32(d.done + blk) != p0.epoch + part) {}
      __syncthreads();
    }
  }
  if (p0.symblk && p0.symblk[blk]) {   // every group of this block was folded by sym2_kernel: only keep the hand-over chain alive
    if (p0.n_parts > 1 && part + 1 < p0.n_parts && threadIdx.x == 0) st_release_u32(d.done + blk, p0.epoch + part + 1);
    return;
  }
  const uint32_t g = blk * GROUPS_PER_CTA + lane;  // padded groups (g >= G) are real, unused replicas
  const bool folded = p0.symdone && p0.symdone[g];   // this lane's group is done: it idles through the barriers
  // Which replica of group g this thread steps.  Plain variant: replica index = warp index, so a
  // warp runs one role's code when the CTA's leaders share a replica index (and every branch on
  // `r` is provably warp-uniform).  SORTED variant, picked by the host when a previous launch saw
  // leaders on several indices: the group's live leader goes to warp 0, the others follow in
  // index order.  Pure scheduling -- state planes and mailboxes are indexed by replica.
  uint32_t r = w;
  if constexpr (SORTED) {
    uint32_t lead = R;
#pragma unroll
    for (int rr = 0; rr < R; ++rr) {
      const uint32_t m = d.p2[(size_t)rr * d.Gp + g].w, role = meta_role(m), fault = meta_fault(m), dead = meta_dead(m);
      if (lead == (uint32_t)R && role == JR_ROLE_LEADER && fault == 0 && !dead) lead = rr;
    }
    if (lead != (uint32_t)R) r = w == 0 ? lead : (w <= lead ? w - 1 : w);
  }
  const uint32_t box = d.Us * R * 32;
  Local L;
  L.in = smem;
  L.out = smem + box;
  L.tc = smem + 2 * box;
  L.cin = reinterpret_cast<uint32_t*>(smem + 2 * box + d.W * R * 32);
  L.cout = L.cin + R * 32;
  L.mk_in = reinterpret_cast<uint16_t*>(L.cout + R * 32);
  L.mk_out = L.mk_in + R * R * 32;
  L.Us = d.Us; L.W = d.W; L.lane = lane;
  Replica<R, SORTED, QUEUES> rep(d, L, r, g);
  rep.now = p.now;
  rep.cur = p.cur;
  rep.load(p.phases & PH_RESET_OUT, p.phases & PH_RESET_FSM, part != 0);
  if (folded) rep.dead = 1;   // never stepped, never stored
  rep.tc_prefetch();
  rep.stage_inbox(p.phases & PH_DRAIN);
#ifdef JR_PROFILE
  for (uint32_t i = threadIdx.x; i < 8 * 3 * 16 * 2; i += blockDim.x) jr_prof_smem()[i] = 0;
#endif
  __syncthreads();
  StepParams q = p;
  for (uint32_t t = 0;; ++t) {
    JR_PROF_T0(tt);
    const uint32_t prole = rep.role == JR_ROLE_LEADER ? JR_ROLE_LEADER : JR_ROLE_FOLLOWER;
    (void)prole;
    rep.clear_marks();
    rep.run_step(q);
    JR_PROF_ADD(prole, 12, tt);
    if (t + 1 == p.n_ticks) break;
    L.cout[r * 32 + lane] = rep.ocnt;
    rep.publish_marks();
    JR_PROF_ADD(prole, 15, tt);
    __syncthreads();
    JR_PROF_ADD(prole, 13, tt);
    // next tick: what was written becomes the inbox
    uint4* tb = L.in; L.in = L.out; L.out = tb;
    uint32_t* tcn = L.cin; L.cin = L.cout; L.cout = tcn;
    uint16_t* tmk = L.mk_in; L.mk_in = L.mk_out; L.mk_out = tmk;
    rep.cur ^= 1;
    rep.ocnt = 0;
    rep.ocnt0 = 0;
    rep.now += p.dt;
    q.now = rep.now;
    q.step_index += 1;
    q.phases = PH_RESET_OUT | PH_DRAIN | PH_PROPOSE | PH_TICK;
    q.proposals = (p.proposals && p.prop_stride) ? p.proposals + (size_t)(t + 1) * p.prop_stride : nullptr;
    q.tok_tick += 1;
  }
  if (!folded) rep.store(part + 1 >= p0.n_parts);
  {  // tell the host whether the next launch should sort: leaders on >= 2 replica indices in this CTA?
    uint32_t* lmask = reinterpret_cast<uint32_t*>(L.tc);  // the table cache is dead now; reuse one word of it
    __syncthreads();
    if (threadIdx.x == 0) *lmask = 0;
    __syncthreads();
    if (!folded && rep.role == JR_ROLE_LEADER && rep.live()) atomicOr(lmask, 1u << r);
    __syncthreads();
    if (threadIdx.x == 0 && (*lmask & (*lmask - 1u))) *(volatile uint32_t*)d.hscat = p0.epoch;   // advisory, read by the host a launch or two later
  }
  if (p0.n_parts > 1 && part + 1 < p0.n_parts) {  // hand the block over to its next part
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) st_release_u32(d.done + blk, p0.epoch + part + 1);
  }
#ifdef JR_PROFILE
  __syncthreads();
  if (d.prof)
    for (uint32_t i = threadIdx.x; i < R * 3 * 16 * 2; i += blockDim.x) {
      const unsigned long long v = jr_prof_smem()[i];
      if (v) atomicAdd(d.prof + (i % (3 * 16 * 2)), v);
    }
#endif
}

// Host-injected commands: one thread per distinct target replica, commands in
// array order.  targets[i] = {group, replica index, first, count}.  No staging.
template <int R>
__global__ void inject_kernel(const Dev d, const StepParams p, const jr_msg* msgs, const uint4* targets,
                              uint32_t n_targets) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  Local L;
  L.in = L.out = L.tc = nullptr; L.cin = L.cout = nullptr; L.mk_in = L.mk_out = nullptr; L.Us = 0; L.W = 0; L.lane = 0;
  if (i >= n_targets) return;
  const uint4 t = targets[i];
  Replica<R> rep(d, L, t.y, t.x);
  rep.now = p.now;
  rep.cur = p.cur;
  rep.load(false, false);
  for (uint32_t k = 0; k < t.w; ++k) {
    const jr_msg* m = msgs + t.z + k;
    Cmd c;
    c.kind = m->kind; c.flag = m->flag ? 1u : 0u; c.node_id = m->node_id; c.block = (uint32_t)m->block;
    c.nblk = m->n_blocks; c.term = m->term; c.last_term = m->last_term;
    if (m->kind == JR_CMD_CLIENT_REQUEST || m->kind == JR_CMD_CLIENT_RESPONSE) {  // Cmd aliases, see raft_device.cuh
      c.term = m->token;
      c.block = ((uint32_t)m->client_kind << 16) | (m->client_id & 0xffffu);
    }
    c.blk_s = 0; c.blk_at = 0; c.host_msg = m;
    rep.apply(c);
  }
  rep.store();
}

// RaftHandle::new for every replica (mod.rs:428-435; follower.rs:68-95; chain.rs:117-153).
__global__ void init_kernel(const Dev d) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t plane = (size_t)d.R * d.Gp;
  if (i >= plane) return;
  const uint32_t r = (uint32_t)(i / d.Gp), g = (uint32_t)(i % d.Gp);
  const uint32_t timeout = election_timeout_draw(d.seed, d.goff + g, r + 1, 0, d.emin, d.emax);
  d.p0[i] = make_uint4(0, 0, 0, 0);
  d.p1[i] = make_uint4(0, 0, timeout, 1);                 // init(): first draw, election_time = 0
  // head 0, commit 0, id_gen 1; a node this engine does not host is inert (the `dead` bit)
  d.p2[i] = make_uint4(0, 0, 1, meta_pack(JR_ROLE_FOLLOWER, 0, 0, 0, ((d.resident >> r) & 1u) ? 0u : 1u, 0));
  d.p3[i] = make_uint4(0, 0, 0, 0);
  d.mk[i] = 0;
  d.cnext[i] = 0;                                         // genesis block 0 -> 0 (chain.rs:139-153)
  d.ctok[i] = 0;
  d.oc[0][i] = 0;
  d.oc[1][i] = 0;
  d.fc[i] = make_uint2(0, 0);
  if (r == 0) d.tb[g] = 0;
  const uint64_t tag = mix64(((d.goff + g) << 8) | (r + 1));
  d.dg[i] = make_uint4((uint32_t)tag, (uint32_t)(tag >> 32), (uint32_t)tag, (uint32_t)(tag >> 32));
  d.cn[i] = make_uint2(0, 0);
}

// Chain::compact for every live replica (chain.rs:239-253).
__global__ void compact_kernel(const Dev d) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t plane = (size_t)d.R * d.Gp;
  if (i >= plane || (uint32_t)(i % d.Gp) >= d.G) return;
  const uint4 c = d.p2[i];
  if (!meta_live(c.w)) return;  // faulted or dead
  bool have = false;
  uint32_t expect = 0;
  const uint32_t floor = d.tb[i % d.Gp];
  for (uint32_t b = c.y; b-- > floor;) {  // ids in [0, commit), descending; nothing is left below the floor (D7)
    if (b - floor >= d.cap) continue;    // (a commit past the window cannot exist: chain_commit needs the block)
    const uint32_t nx = d.cnext[table_row(d, plane, b, i)];
    if (nx == ABSENT) continue;
    if (have && b != expect) d.cnext[table_row(d, plane, b, i)] = ABSENT;
    expect = nx;  // even for a removed block
    have = true;
  }
}

// ---- CTA-wide sum and exclusive scan ------------------------------------------------------------------------------
// The kernels built on these run CTAs of CTA_THREADS threads (fsm_scan_kernel: one CTA of SCAN_THREADS), multiples of 32.
// The CPU emulation (tests/emu) runs a CTA's threads one after another, with no warp shuffles and no barriers, so there
// these kernels run one-thread CTAs, where both primitives are the identity.
#ifdef JR_EMU
constexpr uint32_t CTA_THREADS = 1, SCAN_THREADS = 1;
#else
constexpr uint32_t CTA_THREADS = 256, SCAN_THREADS = 1024;
#endif

struct SumOp { template <class T> __device__ __forceinline__ T operator()(T a, T b) const { return a + b; } };
struct MaxOp { template <class T> __device__ __forceinline__ T operator()(T a, T b) const { return max(a, b); } };

// Combines each of the N values over the CTA's threads; thread 0 ends with the CTA totals in v.  smem: one word per
// value and warp; it may be reused after a __syncthreads().
template <class T, int N, class Op = SumOp>
__device__ __forceinline__ void cta_sum(T (&v)[N], T (&smem)[N][32], Op op = Op()) {
#ifdef JR_EMU
  assert(blockDim.x == 1);
  (void)smem; (void)op;
#else
  const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
#pragma unroll
  for (int c = 0; c < N; ++c) {
    for (int o = 16; o > 0; o >>= 1) v[c] = op(v[c], __shfl_down_sync(0xffffffffu, v[c], o));
    if (lane == 0) smem[c][w] = v[c];
  }
  __syncthreads();
  if (threadIdx.x == 0)
    for (uint32_t k = 1; k < (blockDim.x + 31) / 32; ++k)
#pragma unroll
      for (int c = 0; c < N; ++c) v[c] = op(v[c], smem[c][k]);
#endif
}

// Returns the sum of v over the CTA's threads below this one; *total (if given) = the sum over all of them.  smem: one
// word per warp; it may be reused after a __syncthreads().
template <class T>
__device__ __forceinline__ T cta_exclusive_scan(T v, T* smem, T* total = nullptr) {
#ifdef JR_EMU
  assert(blockDim.x == 1);
  (void)smem;
  if (total) *total = v;
  return 0;
#else
  const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
  T inc = v;
  for (int o = 1; o < 32; o <<= 1) {
    const T x = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= (uint32_t)o) inc += x;
  }
  if (lane == 31) smem[w] = inc;
  __syncthreads();
  T base = 0;
  for (uint32_t k = 0; k < w; ++k) base += smem[k];
  if (total) {
    T t = base;
    for (uint32_t k = w; k < (blockDim.x + 31) / 32; ++k) t += smem[k];
    *total = t;
  }
  return base + inc - v;
#endif
}

// Normative state digest (DESIGN.md "Digests"); must equal jro_state_digest.
__global__ void state_digest_kernel(const Dev d, unsigned long long* out) {
  __shared__ uint64_t sm[1][32];
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t plane = (size_t)d.R * d.Gp;
  uint64_t h = 0;
  if (i < plane && (uint32_t)(i % d.Gp) < d.G) {
    const uint32_t r = (uint32_t)(i / d.Gp), g = (uint32_t)(i % d.Gp);
    const uint4 a = d.p0[i], b = d.p1[i], c = d.p2[i];
    const uint32_t role = meta_role(c.w), fault = meta_fault(c.w), prmask = meta_prmask(c.w);
    const uint32_t nq = meta_nq(c.w), dead = meta_dead(c.w);
    h = mix64(0x243f6a8885a308d3ull ^ (((d.goff + g) << 8) | (r + 1)));
    h = fold(h, (uint64_t)a.x | ((uint64_t)a.y << 32));
    h = fold(h, a.z);
    h = fold(h, (uint64_t)role | ((uint64_t)fault << 8) | ((uint64_t)(dead ? 0 : 1) << 16) | ((uint64_t)nq << 24));
    h = fold(h, (uint64_t)b.x | ((uint64_t)b.y << 32));
    h = fold(h, (uint64_t)b.z | ((uint64_t)b.w << 32));
    h = fold(h, c.x);
    h = fold(h, c.y);
    h = fold(h, c.z);
    if (role == JR_ROLE_FOLLOWER) h = fold(h, a.w);
    if (role == JR_ROLE_CANDIDATE) {
      const uint4 e = d.p3[i];
      h = fold(h, (uint64_t)e.z | ((uint64_t)e.w << 32));
    }
    if (role == JR_ROLE_LEADER) {
      const uint4 e = d.p3[i];
      h = fold(h, (uint64_t)e.x | ((uint64_t)e.y << 32));
      for (uint32_t k = 0; k < d.R; ++k) {
        const uint4 v = d.pr[(size_t)(k / 4) * plane + i];
        const uint32_t ph = (k & 3) == 0 ? v.x : (k & 3) == 1 ? v.y : (k & 3) == 2 ? v.z : v.w;
        h = fold(h, ph);
      }
      h = fold(h, prmask);
    }
    for (uint32_t q = 0; q < nq; ++q) {
      const uint4 e = d.qt[(size_t)q * plane + i];
      h = fold(h, (uint64_t)e.x | ((uint64_t)e.y << 32));
      h = fold(h, (uint64_t)(e.z >> 16) | ((uint64_t)(e.z & 0xffffu) << 8));
    }
    uint64_t chain = 0;
    const uint32_t mk = d.mk[i], floor = d.tb[g];
    for (uint32_t bid = floor; bid <= mk && bid - floor < d.cap; ++bid) {
      const uint32_t nx = d.cnext[table_row(d, plane, bid, i)];
      if (nx == ABSENT) continue;
      const uint64_t tok = d.ctok[table_row(d, plane, bid, i)];
      chain += mix64(mix64((uint64_t)bid + 0x13198a2e03707344ull) ^ ((uint64_t)nx * 0xa4093822299f31d1ull) ^ tok);
    }
    h = fold(h, chain);
  }
  uint64_t v[1] = {h};
  cta_sum(v, sm);
  if (threadIdx.x == 0) atomicAdd(out, (unsigned long long)v[0]);
}

// out[0..3] = sum msg digest, sum fsm digest, n msgs, n fsm; out[4] = faulted replicas
__global__ void stream_digest_kernel(const Dev d, unsigned long long* out) {
  __shared__ uint64_t sm[5][32];
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t plane = (size_t)d.R * d.Gp;
  uint64_t v[5] = {0, 0, 0, 0, 0};
  if (i < plane && (uint32_t)(i % d.Gp) < d.G) {
    const uint4 g = d.dg[i];
    const uint2 n = d.cn[i];
    v[0] = (uint64_t)g.x | ((uint64_t)g.y << 32);
    v[1] = (uint64_t)g.z | ((uint64_t)g.w << 32);
    v[2] = n.x;
    v[3] = n.y;
    v[4] = meta_fault(d.p2[i].w) != 0;
  }
  cta_sum(v, sm);
  if (threadIdx.x == 0)
    for (int c = 0; c < 5; ++c) atomicAdd(out + c, (unsigned long long)v[c]);
}

// Leader::write_state (leader.rs:101-121) for every group: the live leader with
// the highest (term, id).  One thread per group.
__global__ void leader_table_kernel(const Dev d, jr_leader_entry* out, uint32_t* route) {
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= d.G) return;
  jr_leader_entry e{0, 0, 0};
  for (uint32_t r = 0; r < d.R; ++r) {
    const size_t i = (size_t)r * d.Gp + g;
    const uint4 c = d.p2[i];
    if (meta_role(c.w) != JR_ROLE_LEADER || !meta_live(c.w)) continue;
    const uint4 a = d.p0[i];
    const uint64_t term = (uint64_t)a.x | ((uint64_t)a.y << 32);
    if (e.leader_id == 0 || term >= e.term) {
      e.term = term;
      e.leader_id = r + 1;
      e.commit = c.y;
    }
  }
  out[g] = e;
  route[g] = e.leader_id;  // where jr_run_tokens sends this group's proposals until the next announce
}

// jr_run_tokens: tokens[k*G + g] -> jr_proposal{token, node = last announced leader of g}.  Pure streaming
// (8 B in, 16 B out per group-tick); the step kernel then reads the same dense layout jr_run_proposals stages.
__global__ void route_tokens_kernel(const unsigned long long* __restrict__ tokens, const uint32_t* __restrict__ route,
                                    jr_proposal* __restrict__ out, uint32_t G, size_t n) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const unsigned long long t = tokens[i];
    jr_proposal p;
    p.token = t;
    p.node = t ? route[i % G] : 0u;
    p.reserved = 0;
    out[i] = p;
  }
}

__global__ void kill_leaders_kernel(const Dev d, uint64_t base, uint32_t permille, unsigned long long* n_killed) {
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  const bool pick = g < d.G && mix64(base + d.goff + g) % 1000 < permille;
  uint32_t killed = 0;
  for (uint32_t r = 0; r < d.R; ++r) {
    bool hit = false;
    if (pick) {
      const size_t i = (size_t)r * d.Gp + g;
      const uint32_t m = d.p2[i].w;
      hit = meta_role(m) == JR_ROLE_LEADER && meta_live(m);
      if (hit) d.p2[i].w = m | META_DEAD;
    }
#ifdef JR_EMU
    killed += hit ? 1u : 0u;
#else
    // warp-aggregated count: one vote per lane, popcount of the ballot, one atomic per warp
    const uint32_t votes = __ballot_sync(0xffffffffu, hit);
    if ((threadIdx.x & 31u) == 0) killed += (uint32_t)__popc(votes);
#endif
  }
  if (killed) atomicAdd(n_killed, (unsigned long long)killed);
}

// jr_isolate_leaders: kill_leaders_kernel's selection; each live leader of a picked group loses every link to and from it.
__global__ void isolate_leaders_kernel(const Dev d, uint64_t base, uint32_t permille, unsigned long long* n_isolated) {
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  const bool pick = g < d.G && mix64(base + d.goff + g) % 1000 < permille;
  bool hit = false;   // the group has a live leader (at R = 1 it has no link to cut, and still counts)
  if (pick) {
    const unsigned long long row = (1ull << d.R) - 1ull;   // one row: every sender 1..R
    unsigned long long col = 0, m = 0;                      // one column: every receiver 1..R
    for (uint32_t r = 0; r < d.R; ++r) col |= 1ull << (8u * r);
    for (uint32_t r = 0; r < d.R; ++r) {
      const uint32_t meta = d.p2[(size_t)r * d.Gp + g].w;
      if (meta_role(meta) == JR_ROLE_LEADER && meta_live(meta)) {
        m |= (row << (8u * r)) | (col << r);
        hit = true;
      }
    }
    for (uint32_t r = 0; r < d.R; ++r) m &= ~(1ull << (9u * r));   // (the diagonal stays clear)
    if (m) d.links[g] |= m;
  }
#ifdef JR_EMU
  const uint32_t isolated = hit ? 1u : 0u;
#else
  // warp-aggregated count: one vote per lane, popcount of the ballot, one atomic per warp
  const uint32_t votes = __ballot_sync(0xffffffffu, hit);
  const uint32_t isolated = (threadIdx.x & 31u) == 0 ? (uint32_t)__popc(votes) : 0u;
#endif
  if (isolated) atomicAdd(n_isolated, (unsigned long long)isolated);
}

// jr_set_links / jr_get_links with a group list: in = {cuts[0 .. n), groups[0 .. n)}, host-validated.
__global__ void links_scatter_kernel(const Dev d, const unsigned long long* cuts, const uint32_t* groups, uint32_t n) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) d.links[groups[k]] = cuts[k];
}
__global__ void links_gather_kernel(const Dev d, const uint32_t* groups, uint32_t n, unsigned long long* out) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) out[k] = d.links[groups[k]];
}

// jr_get_link_queues: depths[64*k + 8*r + s] = Messages queued on link s -> r of groups[k] (groups null: group k).
__global__ void link_queues_gather_kernel(const Dev d, const uint32_t* groups, uint32_t n, uint8_t* depths) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint32_t g = groups ? groups[k] : k;
  uint8_t* o = depths + 64 * (size_t)k;
  for (uint32_t x = 0; x < 64; ++x) o[x] = 0;
  for (uint32_t r = 0; r < d.R; ++r)
    for (uint32_t s = 0; s < d.R; ++s)
      if (s != r) o[8 * r + s] = (uint8_t)(d.lqc[((size_t)lq_slot(r, s) * d.R + r) * d.Gp + g] & 255u);
}

// After node_restart_kernel emptied the queues from the restarted nodes: each named group's non-empty mask, from its
// counts (a separate launch, so that requests for several nodes of one group never race on the mask).
__global__ void link_queues_mask_kernel(const Dev d, const jr_persisted_chain* reqs, uint32_t n) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint32_t g = reqs[k].group;
  unsigned long long m = 0;
  for (uint32_t r = 0; r < d.R; ++r)
    for (uint32_t s = 0; s < d.R; ++s)
      if (s != r && d.lqc[((size_t)lq_slot(r, s) * d.R + r) * d.Gp + g]) m |= 1ull << (8 * r + s);
  d.lqm[g] = m;   // (every request of group g stores the same value)
}

__global__ void set_alive_kernel(const Dev d, uint32_t g, uint32_t r, int alive) {
  const size_t i = (size_t)r * d.Gp + g;
  const uint32_t m = d.p2[i].w;
  d.p2[i].w = alive ? (m & ~META_DEAD) : (m | META_DEAD);
}

// jr_query_many: thread k reads replica (groups[k], nodes[k] - 1)
__global__ void query_kernel(const Dev d, const uint32_t* groups, const uint32_t* nodes, uint32_t n, jr_replica_state* out) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint32_t g = groups[k], r = nodes[k] - 1u;
  jr_replica_state* o = out + k;
  const size_t plane = (size_t)d.R * d.Gp;
  const size_t i = (size_t)r * d.Gp + g;
  const uint4 a = d.p0[i], b = d.p1[i], c = d.p2[i], e = d.p3[i];
  jr_replica_state s;
  memset(&s, 0, sizeof s);
  s.current_term = (uint64_t)a.x | ((uint64_t)a.y << 32);
  s.voted_for = a.z;
  s.role = meta_role(c.w);
  s.leader_id = s.role == JR_ROLE_FOLLOWER ? a.w : 0;
  s.election_time_ms = (uint64_t)b.x | ((uint64_t)b.y << 32);
  s.election_timeout_ms = b.z;
  s.rng_draws = b.w;
  s.head = c.x;
  s.commit = c.y;
  s.id_gen = c.z;
  s.max_key = d.mk[i];
  s.fault = meta_fault(c.w);
  s.alive = meta_dead(c.w) ? 0 : 1;
  s.n_queued = meta_nq(c.w);
  if (s.role == JR_ROLE_LEADER) {
    s.heartbeat_time_ms = (uint64_t)e.x | ((uint64_t)e.y << 32);
    s.progress_replicate = meta_prmask(c.w);
    for (uint32_t k = 0; k < d.R; ++k) {
      const uint4 v = d.pr[(size_t)(k / 4) * plane + i];
      s.progress_head[k] = (k & 3) == 0 ? v.x : (k & 3) == 1 ? v.y : (k & 3) == 2 ? v.z : v.w;
    }
  }
  if (s.role == JR_ROLE_CANDIDATE) {
    s.votes_seen = e.z;
    s.votes_granted = e.w;
  }
  s.chain_floor = d.tb[g];
  *o = s;
}

// jr_chain_read_many: request q = {group, node - 1, first id, output offset}; one CTA per request
__global__ void chain_read_kernel(const Dev d, const uint4* reqs, const uint32_t* counts, jr_block* out, uint8_t* present) {
  const uint32_t q = blockIdx.x;
  const uint4 rq = reqs[q];
  const uint32_t n = counts[q];
  const size_t plane = (size_t)d.R * d.Gp;
  const size_t i = (size_t)rq.y * d.Gp + rq.x;
  const uint32_t floor = d.tb[rq.x];
  for (uint32_t k = threadIdx.x; k < n; k += blockDim.x) {
    const uint64_t bid = (uint64_t)rq.z + k;
    uint32_t nx = ABSENT;
    if (bid >= floor && bid - floor < d.cap) nx = d.cnext[table_row(d, plane, (uint32_t)bid, i)];
    present[rq.w + k] = nx != ABSENT;
    out[rq.w + k] = jr_block{bid, nx != ABSENT ? nx : 0ull,
                             nx != ABSENT ? d.ctok[table_row(d, plane, (uint32_t)bid, i)] : 0ull};
  }
}

// jr_truncate (deviation D7).  One thread per group: new floor = min(commit over live replicas) - margin, never
// below the old one; every block below it leaves the table of EVERY replica of the group (rows are reused by
// the ids one window further up, so they must read as absent).
__global__ void truncate_kernel(const Dev d, uint32_t margin, const uint8_t* skip) {
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= d.Gp) return;
  if (skip && skip[g]) return;   // truncated by the lane that folded the group (sym2_kernel)
  const size_t plane = (size_t)d.R * d.Gp;
  const uint32_t old = d.tb[g];
  uint32_t lo = 0xFFFFFFFFu;
  for (uint32_t r = 0; r < d.R; ++r) {
    const uint4 c = d.p2[(size_t)r * d.Gp + g];
    if (!meta_live(c.w)) continue;  // faulted or silenced: not waited for
    lo = min(lo, c.y);
  }
  if (lo == 0xFFFFFFFFu) return;
  const uint32_t floor = lo > margin ? lo - margin : 0u;
  if (floor <= old) return;
  for (uint32_t b = old; b < floor && b - old < d.cap; ++b)
    for (uint32_t r = 0; r < d.R; ++r) d.cnext[table_row(d, plane, b, (size_t)r * d.Gp + g)] = ABSENT;
  // a replica that was not waited for (silenced / faulted) may have lost every block it held: an empty table's largest key is 0
  for (uint32_t r = 0; r < d.R; ++r)
    if (d.mk[(size_t)r * d.Gp + g] < floor) d.mk[(size_t)r * d.Gp + g] = 0;
  d.tb[g] = floor;
}

// ---- bulk chain export / node restart ---------------------------------------------------------
// One thread per requested replica, looping over table rows: the tables are [row][replica][group], so a warp of
// group-consecutive requests (node k of every group -- the usual restart) touches each row coalesced.

// The part of replica i's window that can hold blocks: ids [floor, floor + span).  Only inserts raise the largest key
// (truncation zeroes it once the floor passes it), so nothing above it is present.
__device__ __forceinline__ uint32_t window_span(const Dev& d, size_t i, uint32_t floor) {
  const uint32_t mk = d.mk[i];
  return mk < floor ? 0u : min(mk - floor + 1u, d.cap);
}

// jr_chain_export_many, pass 1: target k = {group, node - 1}; its descriptor with the number of blocks present
// (first_block is the host's exclusive scan of those counts).
__global__ void export_count_kernel(const Dev d, const uint2* targets, uint32_t n, jr_persisted_chain* out) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint2 t = targets[k];
  const size_t plane = (size_t)d.R * d.Gp;
  const size_t i = (size_t)t.y * d.Gp + t.x;
  const uint32_t floor = d.tb[t.x], span = window_span(d, i, floor);
  uint32_t cnt = 0;
  for (uint32_t b = 0; b < span; ++b) cnt += d.cnext[table_row(d, plane, floor + b, i)] != ABSENT ? 1u : 0u;
  const uint4 c = d.p2[i];
  jr_persisted_chain o;
  o.group = t.x;
  o.node = t.y + 1;
  o.commit = c.y;
  o.first_block = 0;
  o.n_blocks = cnt;
  o.commit_key = meta_ckey(c.w);
  out[k] = o;
}

// jr_chain_export_many, pass 2: target k's blocks, ascending id, to out[first_block ..].
__global__ void export_pack_kernel(const Dev d, const jr_persisted_chain* desc, uint32_t n, jr_block* out) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const jr_persisted_chain c = desc[k];
  const size_t plane = (size_t)d.R * d.Gp;
  const size_t i = (size_t)(c.node - 1) * d.Gp + c.group;
  const uint32_t floor = d.tb[c.group], span = window_span(d, i, floor);
  jr_block* o = out + c.first_block;
  for (uint32_t b = 0, j = 0; b < span && j < c.n_blocks; ++b) {
    const size_t row = table_row(d, plane, floor + b, i);
    const uint32_t nx = d.cnext[row];
    if (nx != ABSENT) o[j++] = jr_block{(uint64_t)floor + b, nx, d.ctok[row]};
  }
}

// jr_node_restart_many: Chain::new over a persisted tree (chain.rs:117-137) + Raft::<Follower>::new (follower.rs:68-95),
// request k = reqs[k].  Host-validated: distinct replicas; ids strictly ascending inside [floor, floor + cap).  From host
// data the window is emptied (an empty sled tree) and refilled; JR_RESTART_IN_PLACE keeps the rows and takes commit and
// the commit key from the replica's own P2 -- the tree as the old incarnation left it.
// rm (JR_F_CLIENT_RESPONSES, else null): the new process's fsm::Driver starts with an empty map (server.rs:80-81, fsm.rs:48)
// from this point of the replica's Instruction stream on; the next drain's fsm_respond_kernel clears the map there.
__global__ void node_restart_kernel(const Dev d, uint64_t now, const jr_persisted_chain* reqs, uint32_t n, const jr_block* blocks,
                                    uint4* rm) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const jr_persisted_chain q = reqs[k];
  const uint32_t g = q.group, r = q.node - 1;
  const size_t plane = (size_t)d.R * d.Gp;
  const size_t i = (size_t)r * d.Gp + g;
  const uint32_t floor = d.tb[g];
  uint32_t commit, ckey, mk = 0;
  if (q.n_blocks == JR_RESTART_IN_PLACE) {
    const uint4 c = d.p2[i];
    commit = c.y;
    ckey = meta_ckey(c.w);
    for (uint32_t b = window_span(d, i, floor); b-- > 0;)   // the largest key becomes exact, as an export would make it
      if (d.cnext[table_row(d, plane, floor + b, i)] != ABSENT) { mk = floor + b; break; }
  } else {
    commit = (uint32_t)q.commit;
    ckey = q.commit_key ? 1u : 0u;
    for (uint32_t b = 0; b < d.cap; ++b) d.cnext[table_row(d, plane, floor + b, i)] = ABSENT;
    const jr_block* bl = blocks + q.first_block;
    for (uint32_t j = 0; j < q.n_blocks; ++j) {
      const uint32_t bid = (uint32_t)bl[j].id;
      d.cnext[table_row(d, plane, bid, i)] = (uint32_t)bl[j].next;
      d.ctok[table_row(d, plane, bid, i)] = bl[j].data;
      mk = bid;                        // ascending: the last one is the largest
    }
  }
  uint32_t idgen = commit;             // IdGenerator::new(commit), chain.rs:126
  if (commit == 0) {                   // chain.init(), chain.rs:139-153: id_gen.next() == 0, block 0 -> 0 inserted
    if (floor == 0) { d.cnext[i] = 0; d.ctok[i] = 0; }
    idgen = 1;
  }
  const uint32_t timeout = election_timeout_draw(d.seed, d.goff + g, r + 1, 0, d.emin, d.emax);
  d.p0[i] = make_uint4(0, 0, 0, 0);
  d.p1[i] = make_uint4((uint32_t)now, (uint32_t)(now >> 32), timeout, 1);
  d.p2[i] = make_uint4(commit, commit, idgen, meta_pack(JR_ROLE_FOLLOWER, 0, 0, 0, 0, ckey));
  d.p3[i] = make_uint4(0, 0, 0, 0);
  d.mk[i] = mk;
  d.oc[0][i] = 0;
  d.oc[1][i] = 0;
  if (d.lqc)   // a new process has new channels: the queues FROM this node are gone (link_queues_mask_kernel follows)
    for (uint32_t q = 0; q < d.R; ++q)
      if (q != r) d.lqc[((size_t)lq_slot(q, r) * d.R + q) * d.Gp + g] = 0;
  if (rm) {
    const uint32_t pos = d.fc[i].y;
    uint4 m = rm[i];
    if (!m.z) m.x = pos;
    m.y = pos;
    m.z = min(m.z + 1u, 3u);
    rm[i] = m;
  }
}

// jr_step starts every replica's Instruction FIFO afresh: the Instructions before a pending restart are gone, so the map
// is cleared at the start of the new stream.
__global__ void restart_marks_rebase_kernel(const Dev d, uint4* rm) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < (size_t)d.R * d.Gp && rm[i].z) rm[i] = make_uint4(0u, 0u, 1u, 0u);
}

// ---- replica verification (jr_verify_groups; the rules are normative in the ABI header) -------------------------------
// Read-only.  Two passes of one thread per replica of the listed groups, thread t = (node - 1) * n + list index: threads
// are group-consecutive, so a warp over groups that sit at the same ids (steady state) loads each table row coalesced.
//   verify_walk_kernel   the replica's own committed chain -> vw[t] = {verdict, id}
//   verify_judge_kernel  the group's reference from its R verdicts; an intact replica other than the reference walks its
//                        chain against the reference's; leader conflicts; the report's counts -> vf[t]
// Only when there is something to report: verify_count / scan / pack put the findings in (group, node) order.
constexpr uint32_t VW_SKIP = 0, VW_INTACT = 7;   // walk verdicts besides JR_VERIFY_BELOW_FLOOR .. JR_VERIFY_CHAIN_BROKEN
constexpr int VERIFY_COUNTS = 7;                 // jr_verify_report from replicas_checked on

__device__ __forceinline__ uint32_t verify_group(const uint32_t* groups, uint32_t j) { return groups ? groups[j] : j; }

__global__ void verify_walk_kernel(const Dev d, const uint32_t* groups, uint32_t n, uint2* vw) {
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (size_t)d.R * n) return;
  const uint32_t r = (uint32_t)(t / n), g = verify_group(groups, (uint32_t)(t % n));
  const size_t plane = (size_t)d.R * d.Gp, i = (size_t)r * d.Gp + g;
  const uint32_t meta = d.p2[i].w, cm = d.p2[i].y, floor = d.tb[g];
  uint2 v = make_uint2(VW_SKIP, 0u);
  if (meta_live(meta)) {
    if (cm < floor) {
      v = make_uint2(JR_VERIFY_BELOW_FLOOR, cm);
    } else if (cm - floor >= d.cap || d.cnext[table_row(d, plane, cm, i)] == ABSENT) {
      v = make_uint2(JR_VERIFY_COMMIT_ABSENT, cm);
    } else {
      v = make_uint2(VW_INTACT, cm);
      uint32_t x = cm;
      for (uint32_t s = 0; s < d.cap; ++s) {   // ids fall strictly inside [floor, floor + cap): at most cap steps
        const uint32_t nx = d.cnext[table_row(d, plane, x, i)];
        // absent (ABSENT is above every id) or a next that is not below its id, genesis 0 -> 0 excepted
        if (nx >= x && (x | nx) != 0) { v = make_uint2(JR_VERIFY_CHAIN_BROKEN, x); break; }
        if (x == 0 || nx < floor) break;
        x = nx;
      }
    }
  }
  vw[t] = v;
}

// vf[t] = {kind | ref node << 8 | conflict mask << 16, id}: kind 0 = no replica finding; the conflict mask is set on the
// lowest leader of a term two or more checked leaders share.  rep += this CTA's counts (one atomic per count and CTA).
__global__ void verify_judge_kernel(const Dev d, const uint32_t* groups, uint32_t n, const uint2* vw, uint2* vf,
                                    unsigned long long* rep) {
  __shared__ uint64_t s[VERIFY_COUNTS][32];
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint64_t cnt[VERIFY_COUNTS] = {0, 0, 0, 0, 0, 0, 0};   // checked, skipped, below floor, absent, broken, diverged, conflicts
  if (t < (size_t)d.R * n) {
    const uint32_t r = (uint32_t)(t / n), j = (uint32_t)(t % n), g = verify_group(groups, j);
    const size_t plane = (size_t)d.R * d.Gp, i = (size_t)r * d.Gp + g;
    uint32_t ref = 0, refc = 0;   // node id, commit
    for (uint32_t k = 0; k < d.R; ++k) {
      const uint2 w = vw[(size_t)k * n + j];
      if (w.x == VW_INTACT && (ref == 0 || w.y > refc)) { ref = k + 1; refc = w.y; }
    }
    const uint2 mine = vw[t];
    uint32_t kind = mine.x == VW_INTACT ? 0u : mine.x, id = mine.y, lc = 0;
    if (mine.x == VW_INTACT && ref != r + 1) {
      const size_t ir = (size_t)(ref - 1) * d.Gp + g;
      const uint32_t cm = mine.y, floor = d.tb[g];
      uint32_t y = refc;   // down the reference's chain to the first id <= c_n: c_n is on it iff that id is c_n
      for (uint32_t s2 = 0; s2 < d.cap && y > cm; ++s2) y = d.cnext[table_row(d, plane, y, ir)];
      if (y != cm) {
        kind = JR_VERIFY_DIVERGED;
      } else {             // then both chains share every block down to the first row that differs
        uint32_t x = cm;
        for (uint32_t s2 = 0; s2 < d.cap; ++s2) {
          const size_t ri = table_row(d, plane, x, i), rr = table_row(d, plane, x, ir);
          const uint32_t nx = d.cnext[ri];
          if (nx != d.cnext[rr] || d.ctok[ri] != d.ctok[rr]) { kind = JR_VERIFY_DIVERGED; id = x; break; }
          if (x == 0 || nx < floor) break;
          x = nx;
        }
      }
    }
    if (mine.x != VW_SKIP && meta_role(d.p2[i].w) == JR_ROLE_LEADER) {
      const uint32_t term_lo = d.p0[i].x, term_hi = d.p0[i].y;
      for (uint32_t k = 0; k < d.R; ++k) {
        const size_t ik = (size_t)k * d.Gp + g;
        if (vw[(size_t)k * n + j].x != VW_SKIP && meta_role(d.p2[ik].w) == JR_ROLE_LEADER && d.p0[ik].x == term_lo &&
            d.p0[ik].y == term_hi)
          lc |= 1u << k;
      }
      if (__popc(lc) < 2 || (lc & ((1u << r) - 1u))) lc = 0;   // reported once, by the lowest leader of the term
    }
    vf[t] = make_uint2(kind | (ref << 8) | (lc << 16), id);
    cnt[0] = mine.x != VW_SKIP;
    cnt[1] = mine.x == VW_SKIP;
#pragma unroll
    for (int c = 2; c < 6; ++c) cnt[c] = kind == (uint32_t)(c - 1);   // (static indices: the counts stay in registers)
    cnt[6] = lc != 0;
  }
  cta_sum(cnt, s);
  if (threadIdx.x == 0)
    for (int c = 0; c < VERIFY_COUNTS; ++c)
      if (cnt[c]) atomicAdd(rep + c, (unsigned long long)cnt[c]);
}

__device__ __forceinline__ uint32_t verify_findings_of(const Dev& d, const uint2* vf, uint32_t n, uint32_t j) {
  uint32_t c = 0;
  for (uint32_t k = 0; k < d.R; ++k) {
    const uint32_t v = vf[(size_t)k * n + j].x;
    c += ((v & 255u) != 0) + ((v >> 16) != 0);
  }
  return c;
}

// One thread per listed group: part[CTA] = the CTA's findings.
__global__ void verify_count_kernel(const Dev d, uint32_t n, const uint2* vf, unsigned long long* part) {
  __shared__ uint32_t s[1][32];
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t c[1] = {j < n ? verify_findings_of(d, vf, n, j) : 0u};
  cta_sum(c, s);
  if (threadIdx.x == 0) part[blockIdx.x] = c[0];
}

// One thread: exclusive scan of the per-CTA counts (it only runs when some group has findings).
__global__ void verify_scan_kernel(unsigned long long* part, uint32_t n_ctas) {
  unsigned long long at = 0;
  for (uint32_t k = 0; k < n_ctas; ++k) { const unsigned long long v = part[k]; part[k] = at; at += v; }
}

// One thread per listed group: its findings at part[CTA] + the CTA-local exclusive scan -- leader conflicts by their
// lowest leader, then the replica findings by node.
__global__ void verify_pack_kernel(const Dev d, const uint32_t* groups, uint32_t n, const uint2* vf,
                                   const unsigned long long* part, jr_verify_finding* out) {
  __shared__ uint32_t s_warp[32];
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t c = j < n ? verify_findings_of(d, vf, n, j) : 0u;
  const uint32_t pre = cta_exclusive_scan(c, s_warp);
  if (j >= n || c == 0) return;
  const uint32_t g = verify_group(groups, j);
  jr_verify_finding* o = out + part[blockIdx.x] + pre;
  for (int pass = 0; pass < 2; ++pass)
    for (uint32_t k = 0; k < d.R; ++k) {
      const uint2 v = vf[(size_t)k * n + j];
      const uint32_t kind = pass == 0 ? ((v.x >> 16) ? (uint32_t)JR_VERIFY_LEADER_CONFLICT : 0u) : (v.x & 255u);
      if (!kind) continue;
      const uint4 a = d.p0[(size_t)k * d.Gp + g];
      jr_verify_finding f;
      f.group = g;
      f.kind = (uint8_t)kind;
      f.node = pass == 0 ? 0 : (uint8_t)(k + 1);
      f.ref_node = (uint8_t)((v.x >> 8) & 255u);
      f.node_mask = (uint8_t)(pass == 0 ? (v.x >> 16) : (1u << k));
      f.id = pass == 0 ? 0 : v.y;
      f.term = (uint64_t)a.x | ((uint64_t)a.y << 32);
      f.reserved = 0;
      *o++ = f;
    }
}

// ---- Instruction-stream drain -----------------------------------------------------------------
// Records sit in per-replica FIFOs ([2*rec + half][replica][group]).  The drain packs them into one dense
// array in thread order i = replica * Gp + group -- sorted by (node, group), FIFO per replica -- with an exclusive
// scan over the per-replica counts, writes them to a device staging buffer and empties the FIFOs; the copy engine
// takes the batch to pinned host memory (fsm_records_enqueue).
struct FsmHeader {          // written by fsm_pack_kernel next to the records
  unsigned long long n_records, n_dropped, n_instructions;
  uint32_t node_offset[JR_MAX_REPLICAS + 1];
  unsigned long long n_wanted;   // records the FIFOs held, before the cut at the batch's capacity
};

// Three small kernels on cta_sum / cta_exclusive_scan:
//   fsm_count_kernel  per-CTA sums of the replicas' record counts            -> part[3][n_ctas]
//   fsm_scan_kernel   one CTA: exclusive scan of those sums, batch totals     -> part[0] becomes CTA offsets, hdr
//   fsm_pack_kernel   CTA-local scan + CTA offset = each replica's position; copies its records, empties its FIFO
// Padded groups (g >= G) contribute nothing.  The same three pack the client responses (JR_F_CLIENT_RESPONSES): they
// work on the FIFO, counts {stored, elements} and staging they are given, F runs per replica either way.
__device__ __forceinline__ uint32_t fsm_kept(const Dev& d, size_t i, uint2 c) {
  return (uint32_t)(i % d.Gp) < d.G ? min(c.x, d.F) : 0u;
}

// `xdrop` (may be null): elements each replica lost besides the runs beyond F.
__global__ void fsm_count_kernel(const Dev d, const uint2* cnt, const uint32_t* xdrop, unsigned long long* part, uint32_t n_ctas) {
  __shared__ unsigned long long s[3][32];
  const size_t plane = (size_t)d.R * d.Gp;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long v[3] = {0, 0, 0};   // records, dropped, Instructions
  if (i < plane && (uint32_t)(i % d.Gp) < d.G) {
    const uint2 c = cnt[i];
    v[0] = min(c.x, d.F);
    v[1] = (c.x > d.F ? c.x - d.F : 0u) + (xdrop ? xdrop[i] : 0u);
    v[2] = c.y;
  }
  cta_sum(v, s);
  if (threadIdx.x != 0) return;
  part[blockIdx.x] = v[0];
  part[n_ctas + blockIdx.x] = v[1];
  part[2 * (size_t)n_ctas + blockIdx.x] = v[2];
}

// elem_drops: records cut off by cap_records are counted by their elements, in fsm_pack_kernel (the client responses: their
// n_dropped counts responses), instead of one each here.
__global__ void fsm_scan_kernel(unsigned long long* part, uint32_t n_ctas, FsmHeader* hdr, uint32_t cap_records, bool elem_drops) {
  __shared__ unsigned long long s_warp[32];
  const uint32_t t = threadIdx.x, T = blockDim.x;
  const uint32_t per = (n_ctas + T - 1) / T;
  const uint32_t lo = min(n_ctas, per * t), hi = min(n_ctas, per * (t + 1));
  unsigned long long sum = 0, drop = 0, ins = 0;
  for (uint32_t k = lo; k < hi; ++k) { sum += part[k]; drop += part[n_ctas + k]; ins += part[2 * (size_t)n_ctas + k]; }
  unsigned long long total;
  unsigned long long at = cta_exclusive_scan(sum, s_warp, &total);
  if (t == 0) {
    hdr->n_records = min(total, (unsigned long long)cap_records);
    hdr->n_dropped = total > cap_records && !elem_drops ? total - cap_records : 0ull;   // + the per-replica drops, added below
    hdr->n_wanted = total;
    hdr->n_instructions = 0;
  }
  __syncthreads();
  if (drop) atomicAdd(&hdr->n_dropped, drop);
  if (ins) atomicAdd(&hdr->n_instructions, ins);
  for (uint32_t k = lo; k < hi; ++k) { const unsigned long long v = part[k]; part[k] = at; at += v; }
}

// Thread i moves its replica's records to out[position ..] and empties the FIFO.  `out` may be mapped host memory.
__global__ void fsm_pack_kernel(const Dev d, const uint4* fifo, uint2* cnt, const unsigned long long* part, FsmHeader* hdr,
                                uint4* out, uint32_t cap_records, bool elem_drops) {
  __shared__ uint32_t s_warp[32];
  const size_t plane = (size_t)d.R * d.Gp;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t n = i < plane ? fsm_kept(d, i, cnt[i]) : 0u;
  const unsigned long long at64 = part[blockIdx.x] + cta_exclusive_scan(n, s_warp);
  if (i < plane) {
    const uint32_t at = (uint32_t)min(at64, (unsigned long long)cap_records);
    for (uint32_t k = 0; k < n && at + k < cap_records; ++k) {
      out[(size_t)2 * (at + k)] = fifo[(size_t)(2 * k) * plane + i];
      out[(size_t)2 * (at + k) + 1] = fifo[(size_t)(2 * k + 1) * plane + i];
    }
    if (elem_drops && at + n > cap_records) {   // (rare: the batch buffer is full)
      unsigned long long lost = 0;
      for (uint32_t k = cap_records > at ? cap_records - at : 0u; k < n; ++k) lost += fifo[(size_t)(2 * k) * plane + i].y >> 8;
      atomicAdd(&hdr->n_dropped, lost);
    }
    if (i % d.Gp == 0) hdr->node_offset[i / d.Gp] = at;
    if (i + 1 == plane) hdr->node_offset[d.R] = (uint32_t)min(at64 + n, (unsigned long long)cap_records);
    cnt[i] = make_uint2(0, 0);
  }
}

// ---- Client responses (JR_F_CLIENT_RESPONSES): fsm::Driver's notification map on the device ---------------------------
// fsm.rs:57-81 per replica: Notify{block_id, id, address} inserts block_id -> (address, id) (HashMap insert: it
// overwrites); Apply{block} skips block 0 (fsm.rs:61-63), otherwise notifications.remove(block.id) and a hit sends
// ClientResponse{id} to the address (fsm.rs:66-76).  Matching is by block id only (DESIGN.md N5).
// The map lives in the PN plane as at most JR_NOTIFY_RUNS runs per replica, oldest first: run = ids id0 .. id0+count-1,
// one address, request tokens tok0 + k*stride.  Steady state is one run of two or three ids.
struct RespPlanes {
  uint4* pn;        // [2*run + half][replica][group]: {id0, count, addr, 0}, {tok0 lo, hi, stride lo, hi}
  uint32_t* pnc;    // [replica][group]: runs held
  uint4* rs;        // this drain's response runs, jr_fsm_record layout, F per replica: [2*k + half][replica][group]
  uint2* rc;        // [replica][group]: {runs stored, responses they stand for}
  uint32_t* rd;     // [replica][group]: notifications and responses dropped by this drain
  uint4* rm;        // [replica][group]: restarts since the last drain {stream position of the first, of the last, count <= 3}
};

// 16-byte units of the PN allocation: runs, run counts (u32, padded), restart marks
inline size_t pn_units(size_t plane) { return 2 * (size_t)JR_NOTIFY_RUNS * plane + (plane + 3) / 4 + plane; }

struct PnRun {
  uint32_t id0, count, addr;
  unsigned long long tok0, stride;
};

// The walk follows jr_fsm_expand: a replica's Apply stream is the masked APPLY records naming it (any replica's FIFO,
// ascending FIFO, in front) and then its own unmasked APPLY records; its Notify stream is its own NOTIFY records; its
// PATTERN records place the Notifies.  One thread per replica; the FIFOs are only read (the pack that empties them runs
// after this kernel).  A replica whose batch lost records -- own FIFO full, a masked record lost in a peer's FIFO (the
// records it can see stand for fewer Instructions than it emitted) or a full batch buffer -- clears its map instead.
// Restarts (rm): a restarted replica's undrained Instructions are still drained, but they belong to the old process's
// Driver, whose map dies with it (server.rs:80-81, fsm.rs:48).  The walk clears the map at the stream position where the
// restart happened: what came before went through the old map, what comes after goes through the new one.  Two restarts
// in one drain are exact as well; with three or more, the Instructions between the first and the last restart are not
// matched at all (their Notifies count as dropped).
__global__ void fsm_respond_kernel(const Dev d, const RespPlanes q, const FsmHeader* hdr, uint32_t cap_records) {
  const size_t plane = (size_t)d.R * d.Gp;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= plane) return;
  const uint32_t r = (uint32_t)(i / d.Gp), g = (uint32_t)(i % d.Gp);
  q.rc[i] = make_uint2(0u, 0u);
  q.rd[i] = 0u;
  if (g >= d.G) return;
  const uint4 m = q.rm[i];
  if (m.z) q.rm[i] = make_uint4(0u, 0u, 0u, 0u);
  const uint2 c = d.fc[i];
  const uint32_t own = min(c.x, d.F);
  uint32_t n = q.pnc[i];
  bool notifies = false;
  for (uint32_t k = 0; k < own && !notifies; ++k) notifies = (d.fs[(size_t)(2 * k) * plane + i].y & 3u) == FSR_NOTIFY;
  if (n == 0 && !notifies) return;   // nothing to match, nothing to insert: every steady-state follower
  auto rec_hdr = [&](uint32_t src, uint32_t k) { return d.fs[(size_t)(2 * k) * plane + (size_t)src * d.Gp + g]; };
  auto u64 = [](uint32_t lo, uint32_t hi) { return (unsigned long long)lo | ((unsigned long long)hi << 32); };
  auto kept =[&](uint32_t src) { return min(d.fc[(size_t)src * d.Gp + g].x, d.F); };
  auto mine = [&](uint32_t src_phase, uint4 h) {   // src_phase < R: masked phase over FIFO src_phase; == R: own records
    const bool apply = (h.y & 3u) == FSR_APPLY;
    return src_phase < d.R ? (apply && h.w != 0u && ((h.w >> r) & 1u)) : (apply && h.w == 0u);
  };
  PnRun t[JR_NOTIFY_RUNS + 1];
  for (uint32_t k = 0; k < n; ++k) {
    const uint4 a = q.pn[(size_t)(2 * k) * plane + i], b = q.pn[(size_t)(2 * k + 1) * plane + i];
    t[k] = PnRun{a.x, a.y, a.z, u64(b.x, b.y), u64(b.z, b.w)};
  }
  uint32_t drop = 0;
  // Instructions the visible records stand for
  unsigned long long seen = 0;
  for (uint32_t src = 0; src <= d.R; ++src) {
    const uint32_t from = src < d.R ? src : r, m = kept(from);
    for (uint32_t k = 0; k < m; ++k) {
      const uint4 h = rec_hdr(from, k);
      if (mine(src, h) || (src == d.R && (h.y & 3u) == FSR_NOTIFY)) seen += h.y >> 8;
    }
  }
  if (c.x > d.F || seen != c.y || hdr->n_wanted > cap_records) {
    for (uint32_t k = 0; k < n; ++k) drop += t[k].count;
    q.pnc[i] = 0u;
    q.rd[i] = drop;
    return;
  }
  auto erase = [&](uint32_t k) {
    for (uint32_t j = k; j + 1 < n; ++j) t[j] = t[j + 1];
    --n;
  };
  auto fit = [&]() {   // over JR_NOTIFY_RUNS: the oldest run goes
    if (n > JR_NOTIFY_RUNS) { drop += t[0].count; erase(0); }
  };
  auto find = [&](uint32_t id) {
    uint32_t k = 0;
    while (k < n && id - t[k].id0 >= t[k].count) ++k;
    return k;
  };
  // notifications.remove(id) of the entry known to sit in run k: its address and request token
  auto take = [&](uint32_t k, uint32_t id, uint32_t& addr, unsigned long long& tok) {
    PnRun& x = t[k];
    const uint32_t off = id - x.id0;
    addr = x.addr;
    tok = x.tok0 + (unsigned long long)off * x.stride;
    if (x.count == 1u) {
      erase(k);
    } else if (off == 0u) {
      x.id0 += 1u; x.tok0 += x.stride; x.count -= 1u;
    } else if (off == x.count - 1u) {
      x.count -= 1u;
    } else {   // split: the ids above `id` become a run of their own, just as old
      const PnRun y{id + 1u, x.count - off - 1u, x.addr, x.tok0 + (unsigned long long)(off + 1u) * x.stride, x.stride};
      x.count = off;
      for (uint32_t j = n; j > k + 1u; --j) t[j] = t[j - 1u];
      t[k + 1u] = y;
      ++n;
      fit();
    }
  };
  // response runs of this drain: the open one extends while block ids, address and tokens continue it
  PnRun o{0u, 0u, 0u, 0ull, 0ull};
  uint32_t n_runs = 0, n_resp = 0;
  auto close = [&]() {
    if (!o.count) return;
    if (n_runs < d.F) {
      q.rs[(size_t)(2 * n_runs) * plane + i] = make_uint4(g, JR_FSMR_RESPONSE | (r << 2) | (o.count << 8), o.id0, o.addr);
      const unsigned long long st = o.count > 1u ? o.stride : 0ull;
      q.rs[(size_t)(2 * n_runs + 1) * plane + i] =
          make_uint4((uint32_t)o.tok0, (uint32_t)(o.tok0 >> 32), (uint32_t)st, (uint32_t)(st >> 32));
      ++n_runs;
      n_resp += o.count;
    } else {
      drop += o.count;
    }
    o.count = 0u;
  };
  // cursors: Apply (phase = source FIFO, then R = own records), Notify, PATTERN window
  uint32_t a_src = 0, a_k = 0, a_e = 0, a_cnt = 0, a_id0 = 0;
  uint32_t n_k = 0, n_e = 0, n_cnt = 0;
  uint4 n_h = make_uint4(0u, 0u, 0u, 0u);
  unsigned long long n_tok0 = 0, n_st = 0;
  uint32_t p_k = 0, w0 = 0, wn = 0, wb2 = 0;
  unsigned long long wb0 = 0, wb1 = 0;
  for (uint32_t pos = 0; pos <= c.y; ++pos) {
    if (m.z && (pos == m.x || pos == m.y)) n = 0u;   // a restart: the new process's Driver starts with an empty map
    if (pos == c.y) break;
    const bool skip = m.z > 2u && pos >= m.x && pos < m.y;
    while (pos >= w0 + wn && p_k < own) {   // the next PATTERN window (they come in stream order)
      const uint4 h = rec_hdr(r, p_k);
      if ((h.y & 3u) == FSR_PATTERN) {
        const uint4 v = d.fs[(size_t)(2 * p_k + 1) * plane + i];
        w0 = h.z; wn = h.y >> 8; wb2 = h.w;
        wb0 = u64(v.x, v.y);
        wb1 = u64(v.z, v.w);
      }
      ++p_k;
    }
    const uint32_t b = pos - w0;
    const bool note = pos >= w0 && b < wn && ((b < 64u ? wb0 >> b : b < 128u ? wb1 >> (b - 64u) : (unsigned long long)(wb2 >> (b - 128u))) & 1ull);
    if (note) {
      while (n_e >= n_cnt && n_k < own) {   // the next NOTIFY record of this replica
        n_h = rec_hdr(r, n_k);
        if ((n_h.y & 3u) == FSR_NOTIFY) {
          const uint4 v = d.fs[(size_t)(2 * n_k + 1) * plane + i];
          n_tok0 = u64(v.x, v.y);
          n_st = u64(v.z, v.w);
          n_cnt = n_h.y >> 8;
          n_e = 0;
        }
        ++n_k;
      }
      if (n_e >= n_cnt) break;   // (a malformed stream; jr_fsm_expand rejects it too)
      const uint32_t id = n_h.z + n_e, addr = n_h.w;
      const unsigned long long tok = n_tok0 + (unsigned long long)n_e * n_st;
      ++n_e;
      if (skip) { ++drop; continue; }
      const uint32_t k = find(id);   // insert overwrites (fsm.rs:80)
      if (k < n) { uint32_t a2; unsigned long long t2; take(k, id, a2, t2); }
      PnRun* last = n ? &t[n - 1u] : nullptr;
      if (last && id == last->id0 + last->count && addr == last->addr && last->count < FS_MAX_RUN &&
          (last->count == 1u || tok == last->tok0 + (unsigned long long)last->count * last->stride)) {
        if (last->count == 1u) last->stride = tok - last->tok0;
        last->count += 1u;
      } else {
        t[n++] = PnRun{id, 1u, addr, tok, 0ull};
        fit();
      }
    } else {
      while (a_e >= a_cnt && a_src <= d.R) {   // the next APPLY record of this replica's stream
        const uint32_t from = a_src < d.R ? a_src : r;
        if (a_k >= kept(from)) { ++a_src; a_k = 0; continue; }
        const uint4 h = rec_hdr(from, a_k++);
        if (mine(a_src, h)) { a_id0 = h.z; a_cnt = h.y >> 8; a_e = 0; }
      }
      if (a_e >= a_cnt) break;
      const uint32_t id = a_id0 + a_e++;
      if (id == 0u || skip) continue;   // fsm.rs:61-63
      const uint32_t k = find(id);
      if (k == n) continue;
      uint32_t addr;
      unsigned long long tok;
      take(k, id, addr, tok);
      if (o.count && id == o.id0 + o.count && addr == o.addr && o.count < FS_MAX_RUN &&
          (o.count == 1u || tok == o.tok0 + (unsigned long long)o.count * o.stride)) {
        if (o.count == 1u) o.stride = tok - o.tok0;
        o.count += 1u;
      } else {
        close();
        o = PnRun{id, 1u, addr, tok, 0ull};
      }
    }
  }
  close();
  for (uint32_t k = 0; k < n; ++k) {
    q.pn[(size_t)(2 * k) * plane + i] = make_uint4(t[k].id0, t[k].count, t[k].addr, 0u);
    q.pn[(size_t)(2 * k + 1) * plane + i] = make_uint4((uint32_t)t[k].tok0, (uint32_t)(t[k].tok0 >> 32), (uint32_t)t[k].stride,
                                                       (uint32_t)(t[k].stride >> 32));
  }
  q.pnc[i] = n;
  q.rc[i] = make_uint2(n_runs, n_resp);
  q.rd[i] = drop;
}

// ---- group export / import (jr_group_export / jr_group_import; the rules are normative in the ABI header) ------------
// An image body holds, per (replica, listed group) in thread order t = (node - 1) * n + list index -- group-consecutive, so
// a warp over consecutive groups reads each table row coalesced -- one fixed record of rec_units 16-byte units: the counts
// {table rows, mailbox units, Instruction records, notification runs}, then the words of every plane the engine's plane
// list (engine_planes, host side) carries word for word.  The variable parts follow, in the same order: the rows present
// in the window as {id, next, token lo, token hi}, ascending id; the previous step's mailbox units; the records (2 units
// each); the notification runs (2 units each).
struct ImgPlane {
  uint32_t* p;      // the plane, as 32-bit words
  uint32_t words;   // words per entry
  uint32_t depth;   // entries per replica (or group), one plane apart
  uint32_t group;   // 1: one entry per group, indexed by the group (TB, the route); else per replica
};

__device__ __forceinline__ uint32_t img_var_units(uint4 c) { return c.x + c.y + 2u * c.z + 2u * c.w; }

// Pass 1: thread t's counts -> cnt[t]; part[CTA] = the CTA's variable units (the host scans them).
__global__ void group_count_kernel(const Dev d, const uint32_t* groups, uint32_t n, int prev, const uint32_t* pnc, uint4* cnt,
                                   unsigned long long* part) {
  __shared__ unsigned long long s[1][32];
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long v[1] = {0};
  if (t < (size_t)d.R * n) {
    const uint32_t r = (uint32_t)(t / n), g = groups[t % n];
    const size_t plane = (size_t)d.R * d.Gp, i = (size_t)r * d.Gp + g;
    const uint32_t floor = d.tb[g], span = window_span(d, i, floor);
    uint32_t rows = 0;
    for (uint32_t b = 0; b < span; ++b) rows += d.cnext[table_row(d, plane, floor + b, i)] != ABSENT ? 1u : 0u;
    const uint32_t recs = (d.flags & JR_F_CAPTURE_FSM) ? min(d.fc[i].x, d.F) : 0u;
    const uint4 c = make_uint4(rows, d.oc[prev][i], recs, pnc ? pnc[i] : 0u);
    cnt[t] = c;
    v[0] = img_var_units(c);
  }
  cta_sum(v, s);
  if (threadIdx.x == 0) part[blockIdx.x] = v[0];
}

// Pass 2: thread t packs its fixed record and, at part[CTA] + the CTA-local scan, its variable part; then detaches the
// replica: silenced, Instruction FIFO, notification map and restart marks empty.  Each thread reads and writes only its own
// replica's column.
__global__ void group_pack_kernel(const Dev d, const uint32_t* groups, uint32_t n, int prev, const ImgPlane* planes,
                                  uint32_t n_planes, uint32_t rec_units, const uint4* cnt, const unsigned long long* part,
                                  uint4* out, const RespPlanes q) {
  __shared__ unsigned long long s_warp[32];
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool mine = t < (size_t)d.R * n;
  const uint4 c = mine ? cnt[t] : make_uint4(0u, 0u, 0u, 0u);
  const unsigned long long at = part[blockIdx.x] + cta_exclusive_scan((unsigned long long)img_var_units(c), s_warp);
  if (!mine) return;
  const uint32_t r = (uint32_t)(t / n), g = groups[t % n];
  const size_t plane = (size_t)d.R * d.Gp, i = (size_t)r * d.Gp + g;
  uint4* rec = out + t * rec_units;
  rec[0] = c;
  uint32_t* w = reinterpret_cast<uint32_t*>(rec + 1);
  for (uint32_t k = 0; k < n_planes; ++k) {
    const ImgPlane pl = planes[k];
    const size_t at_p = pl.group ? g : i, stride = pl.group ? d.Gp : plane;
    for (uint32_t e = 0; e < pl.depth; ++e)
      for (uint32_t x = 0; x < pl.words; ++x) *w++ = pl.p[((size_t)e * stride + at_p) * pl.words + x];
  }
  uint4* v = out + (size_t)d.R * n * rec_units + at;
  const uint32_t floor = d.tb[g], span = window_span(d, i, floor);
  for (uint32_t b = 0, k = 0; b < span && k < c.x; ++b) {
    const size_t row = table_row(d, plane, floor + b, i);
    const uint32_t nx = d.cnext[row];
    if (nx == ABSENT) continue;
    const unsigned long long tok = d.ctok[row];
    *v++ = make_uint4(floor + b, nx, (uint32_t)tok, (uint32_t)(tok >> 32));
    ++k;
  }
  for (uint32_t u = 0; u < c.y; ++u) *v++ = d.ob[prev][(size_t)u * plane + i];
  for (uint32_t k = 0; k < 2u * c.z; ++k) *v++ = d.fs[(size_t)k * plane + i];
  for (uint32_t k = 0; k < 2u * c.w; ++k) *v++ = q.pn[(size_t)k * plane + i];
  d.p2[i].w = d.p2[i].w | META_DEAD;
  d.fc[i] = make_uint2(0u, 0u);
  if (q.pnc) {
    q.pnc[i] = 0u;
    q.rm[i] = make_uint4(0u, 0u, 0u, 0u);
  }
}

// Import: one thread per listed group j, into slot slots[j].  Host-validated: distinct slots; counts within the engine's
// limits; rows ascending inside [floor, floor + cap).  The old occupant's rows are only its window_span (truncation keeps
// every other row absent): those are cleared first, then the carried rows, planes, mail, records and runs are written.
// Records carry their group: it becomes the slot.
__global__ void group_unpack_kernel(const Dev d, const uint32_t* slots, uint32_t n, int prev, const ImgPlane* planes,
                                    uint32_t n_planes, uint32_t rec_units, const uint4* img, const unsigned long long* off,
                                    const RespPlanes q) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const uint32_t g = slots[j];
  const size_t plane = (size_t)d.R * d.Gp;
  const uint32_t old_floor = d.tb[g];
  const uint4* var0 = img + (size_t)d.R * n * rec_units;
  for (uint32_t r = 0; r < d.R; ++r) {
    const size_t t = (size_t)r * n + j, i = (size_t)r * d.Gp + g;
    for (uint32_t b = window_span(d, i, old_floor); b-- > 0;) d.cnext[table_row(d, plane, old_floor + b, i)] = ABSENT;
    const uint4* rec = img + t * rec_units;
    const uint4 c = rec[0];
    const uint32_t* w = reinterpret_cast<const uint32_t*>(rec + 1);
    for (uint32_t k = 0; k < n_planes; ++k) {
      const ImgPlane pl = planes[k];
      if (pl.group && r != 0) { w += pl.depth * pl.words; continue; }   // a group's words are taken from its first replica
      const size_t at_p = pl.group ? g : i, stride = pl.group ? d.Gp : plane;
      for (uint32_t e = 0; e < pl.depth; ++e)
        for (uint32_t x = 0; x < pl.words; ++x) pl.p[((size_t)e * stride + at_p) * pl.words + x] = *w++;
    }
    const uint4* v = var0 + off[t];
    for (uint32_t k = 0; k < c.x; ++k, ++v) {
      const size_t row = table_row(d, plane, v->x, i);
      d.cnext[row] = v->y;
      d.ctok[row] = (unsigned long long)v->z | ((unsigned long long)v->w << 32);
    }
    for (uint32_t u = 0; u < c.y; ++u) d.ob[prev][(size_t)u * plane + i] = *v++;
    d.oc[prev][i] = c.y;
    for (uint32_t k = 0; k < c.z; ++k) {
      uint4 h = *v++;
      h.x = g;
      d.fs[(size_t)(2 * k) * plane + i] = h;
      d.fs[(size_t)(2 * k + 1) * plane + i] = *v++;
    }
    for (uint32_t k = 0; k < 2u * c.w; ++k) q.pn[(size_t)k * plane + i] = *v++;
  }
}

__global__ void max_u32_kernel(const uint32_t* v, size_t n, uint32_t* out) {
  __shared__ uint32_t s[1][32];
  uint32_t m[1] = {0};
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    m[0] = max(m[0], v[i]);
  cta_sum(m, s, MaxOp());
  if (threadIdx.x == 0) atomicMax(out, m[0]);
}

// ============================================================================
// host side
// ============================================================================

extern "C" { static jr_status stream_sums(jr_engine* e, uint64_t v[5]); }
static thread_local char g_err[512] = "";
static void set_err(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof g_err, fmt, ap);
  va_end(ap);
}

#define CK(call)                                                                      \
  do {                                                                                \
    cudaError_t _e = (call);                                                          \
    if (_e != cudaSuccess) {                                                          \
      set_err("%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(_e));     \
      return JR_E_CUDA;                                                               \
    }                                                                                 \
  } while (0)

struct jr_engine {
  jr_config cfg;
  Dev d;
  cudaStream_t stream = nullptr;
  cudaStream_t own_stream = nullptr;
  volatile uint32_t* h_scatter = nullptr;  // pinned + mapped: epoch of the last launch that saw scattered leaders (written by the kernel)
  volatile uint32_t* h_unfolded = nullptr; // pinned + mapped: epoch of the last launch whose fold left some group to step_kernel (0: never)
  uint32_t ticket_sum = 0;                 // tickets taken so far (the counter is never reset: each launch gets its base)
  int force_sorted = 0;      // JR_STEP_VARIANT=sorted|plain pins the kernel variant (tests, A/B)
  uint64_t launches_sorted = 0, launches_total = 0, launches_split = 0;
  uint32_t slots = 0;        // CTAs of the step kernel the device holds at once (occupancy x SMs)
  uint32_t sms = 0;          // SMs of the device
  uint32_t force_parts = 0;  // JR_PARTS=n pins the split (tests, A/B); 0 = choose_parts
  int cur = 0;               // outbox index the NEXT step writes
  uint64_t step_index = 0;
  std::vector<void*> allocs;
  // scratch
  unsigned long long* scratch = nullptr;  // 8 x u64 (device)
  jr_msg* inj_msgs = nullptr;             // device, grows
  uint4* inj_targets = nullptr;
  size_t inj_cap = 0;
  // Copy/compute overlap for the host-buffer path: proposals are staged H2D on `h2d`,
  // leader tables leave D2H on `d2h`, both double buffered and fenced with events, so the
  // copy-in of tick k+1, the kernels of tick k and the copy-out of tick k-1 run concurrently.
  static constexpr int NBUF = JR_STAGING_DEPTH;   // staging depth: a host may keep three steps in flight (copy-out, host fold and the next submit overlap)
  jr_proposal* prop[NBUF] = {nullptr, nullptr};         // device, G entries each
  jr_leader_entry* leaders[NBUF] = {nullptr, nullptr};  // device, G entries each
  cudaStream_t h2d = nullptr, d2h = nullptr;
  cudaEvent_t prop_ready[NBUF] = {nullptr, nullptr};    // H2D of prop[i] finished
  cudaEvent_t prop_free[NBUF] = {nullptr, nullptr};     // the kernel that read prop[i] finished
  cudaEvent_t tab_ready[NBUF] = {nullptr, nullptr};     // leader_table_kernel into leaders[i] finished
  cudaEvent_t tab_free[NBUF] = {nullptr, nullptr};      // D2H of leaders[i] finished
  bool prop_used[NBUF] = {false, false}, tab_used[NBUF] = {false, false};
  jr_proposal* batch[NBUF] = {nullptr, nullptr};        // device, batch_cap entries each (jr_run_proposals)
  size_t batch_cap[NBUF] = {0, 0};
  cudaEvent_t batch_ready[NBUF] = {nullptr, nullptr}, batch_free[NBUF] = {nullptr, nullptr};
  bool batch_used[NBUF] = {false, false};
  int batch_i = 0;
  unsigned long long* tokbuf[NBUF] = {nullptr, nullptr};  // device staging of jr_run_tokens input, tok_cap entries each
  size_t tok_cap[NBUF] = {0, 0};
  uint32_t* route = nullptr;              // device, G entries: leader_id of the last leader-table call (0 = none)
  int tab_pending[NBUF] = {0, 0};  // FIFO of leaders[] buffers whose copy-out has not been waited for
  int tab_npending = 0;
  int prop_i = 0, tab_i = 0;
  // scratch of the *_many introspection calls (device, grows)
  void* many_buf = nullptr;
  size_t many_cap = 0;
  // scratch of jr_verify_groups (device, grows; not part of a checkpoint): report, CTA offsets, group list, verdicts
  void* verify_buf = nullptr;
  size_t verify_cap = 0;
  // scratch of jr_group_export / jr_group_import (device, grows; not part of a checkpoint): list, plane list, counts and
  // CTA offsets in move_buf, the image body in move_img
  void* move_buf = nullptr;
  size_t move_cap = 0;
  void* move_img = nullptr;
  size_t move_img_cap = 0;
  // Instruction-stream drain (JR_F_CAPTURE_FSM): scan -> pack into stage[b] on the engine stream, then
  // the copy engine moves stage[b] into the pinned host buffer host[b] on the d2h stream.
  // One slot more than batches may be outstanding, used round robin: with NBUF batches outstanding at a
  // jr_fsm_records_wait, the next enqueue goes to the spare slot, so the batch just returned is reused no earlier
  // than the second enqueue after the wait (the lifetime the ABI header promises), and never while its take runs.
  static constexpr int NSLOT = NBUF + 1;
  unsigned long long* fsm_part = nullptr;                     // device, 3 x (CTAs of the count/pack kernels): per-CTA sums -> offsets
  uint32_t fsm_cap = 0;                                       // records per batch
  uint4* fsm_stage[NSLOT] = {};                               // device, 2 * fsm_cap uint4 each
  FsmHeader* fsm_stage_hdr[NSLOT] = {};                       // device
  uint4* fsm_host[NSLOT] = {};                                // pinned + mapped host
  FsmHeader* fsm_host_hdr[NSLOT] = {};                        // pinned + mapped host
  cudaEvent_t fsm_packed[NSLOT] = {};                         // pack into stage[b] finished (engine stream)
  cudaEvent_t fsm_landed[NSLOT] = {};                         // copy into host[b] finished (d2h stream)
  size_t fsm_copied[NSLOT] = {};                              // records of stage[b] the enqueued copy covers
  size_t fsm_last_records = 0;                                // size of the last batch taken (the next copy's guess)
  bool fsm_used[NSLOT] = {};
  int fsm_i = 0, fsm_pending[NBUF] = {0, 0}, fsm_npending = 0;   // at most NBUF batches outstanding
  std::mutex qmu;   // the two FIFOs of outstanding copy-outs (fsm_pending, tab_pending) and fsm_last_records: a second host thread may
                    // sit in jr_fsm_records_wait / jr_leader_table_wait while the first one keeps submitting
  // client responses (JR_F_CLIENT_RESPONSES): packed into the second region of stage[b] / host[b] (resp_cap records from
  // record fsm_cap on) with their header at fsm_stage_hdr[b][1] / fsm_host_hdr[b][1]
  RespPlanes rp = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  uint32_t resp_cap = 0;
  size_t resp_copied[NSLOT] = {};
  size_t resp_last = 0;                                       // size of the last response batch taken (the next copy's guess)
  int resp_b = -1;                                            // buffer of the batch most recently taken (-1: none yet)
  // symmetric-group fold
  uint8_t* symdone = nullptr;   // device, Gp entries
  uint8_t* symblk = nullptr;    // device, Gp / 32 entries
  uint32_t* symrec = nullptr;   // device, sym_record_words(R) x Gp: sym_check_kernel's entry records (transient, see sym_fold.cuh)
  bool auto_trunc = false;      // jr_set_auto_truncate
  uint32_t auto_trunc_margin = 0;
  int no_fold = 0;              // JR_NO_FOLD=1 (A/B, tests)
  uint64_t launches_folded = 0;
  bool last_launch_folded = false;
};

template <typename T>
static jr_status dalloc(jr_engine* e, T** p, size_t n) {
  void* q = nullptr;
  cudaError_t err = cudaMalloc(&q, n * sizeof(T));
  if (err != cudaSuccess) {
    set_err("cudaMalloc(%zu bytes): %s", n * sizeof(T), cudaGetErrorString(err));
    return err == cudaErrorMemoryAllocation ? JR_E_NOMEM : JR_E_CUDA;
  }
  e->allocs.push_back(q);
  *p = (T*)q;
  return JR_OK;
}

#define DISPATCH_R(R_, CALL)           \
  switch (R_) {                        \
    case 1: { constexpr int RR = 1; CALL; } break; \
    case 2: { constexpr int RR = 2; CALL; } break; \
    case 3: { constexpr int RR = 3; CALL; } break; \
    case 4: { constexpr int RR = 4; CALL; } break; \
    case 5: { constexpr int RR = 5; CALL; } break; \
    case 6: { constexpr int RR = 6; CALL; } break; \
    case 7: { constexpr int RR = 7; CALL; } break; \
    default: { constexpr int RR = 8; CALL; } break; \
  }

// (R = 1 has no links: its engines never need the queue instantiation)
template <int R>
static void launch_step_r(jr_engine* e, const StepParams& p, bool sorted, uint32_t grid, size_t smem) {
  auto kfn = sorted ? step_kernel<R, true> : step_kernel<R, false>;
  if constexpr (R > 1)
    if (e->d.lq) kfn = sorted ? step_kernel<R, true, true> : step_kernel<R, false, true>;
  JR_LAUNCH_SMEM(kfn, grid, 32 * R, smem, e->stream, e->d, p);
}

template <int R>
static cudaError_t step_smem_attr_r(int smem, bool queues) {
  cudaError_t a = cudaFuncSetAttribute(step_kernel<R, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (a == cudaSuccess) a = cudaFuncSetAttribute(step_kernel<R, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if constexpr (R > 1)
    if (queues && a == cudaSuccess) {
      a = cudaFuncSetAttribute(step_kernel<R, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
      if (a == cudaSuccess) a = cudaFuncSetAttribute(step_kernel<R, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    }
  return a;
}

#ifndef JR_EMU
template <int R>
static cudaError_t step_occupancy_r(int* per_sm, int smem) {
  return cudaOccupancyMaxActiveBlocksPerMultiprocessor(per_sm, step_kernel<R, false>, 32 * R, (size_t)smem);
}
#endif

static size_t step_smem_bytes(const Dev& d) {
  return ((size_t)2 * d.Us + d.W) * d.R * 32 * sizeof(uint4) + (size_t)2 * d.R * 32 * sizeof(uint32_t) +
         (size_t)2 * d.R * d.R * 32 * sizeof(uint16_t);
}

// How many consecutive tasks to cut each block's ticks into: the fewest that minimise the number of
// rounds the CTA slots need, in units of a whole-launch task.  1 when the grid fits the slots anyway,
// when the launch is short, or when its first tick is not a whole tick (jr_step's split phases).
static uint32_t choose_parts(const jr_engine* e, const StepParams& p, uint32_t n_blocks) {
  const uint32_t whole = PH_RESET_OUT | PH_DRAIN | PH_TICK;
  if ((p.phases & whole) != whole || p.n_ticks < 2) return 1;
  if (e->force_parts) return std::min<uint32_t>(e->force_parts, p.n_ticks);
  if (!e->slots || n_blocks <= e->slots) return 1;
  uint32_t best = 1;
  double best_rounds = (double)((n_blocks + e->slots - 1) / e->slots);
  for (uint32_t n = 2; n <= 8 && p.n_ticks / n >= 8; n *= 2) {
    const double rounds = (double)(((size_t)n_blocks * n + e->slots - 1) / e->slots) / n;
    if (rounds < best_rounds * 0.97) { best = n; best_rounds = rounds; }
  }
  return best;
}

static jr_status launch_step_once(jr_engine* e, const StepParams& p_in);

// A capturing engine keeps every launch short enough for the raw Instruction FIFO (Fr entries per replica, encoded when
// the launch ends): at most Fr / 3 ticks per launch.  Consecutive launches are indistinguishable from one long launch.
static jr_status launch_step(jr_engine* e, const StepParams& p_in) {
  const uint32_t limit = (e->d.flags & JR_F_CAPTURE_FSM) ? std::max(1u, e->d.Fr / 3u) : 0xffffffffu;
  if (p_in.n_ticks <= limit) return launch_step_once(e, p_in);
  StepParams p = p_in;
  for (uint32_t done = 0; done < p_in.n_ticks;) {
    p.n_ticks = std::min(limit, p_in.n_ticks - done);
    p.trunc = (p_in.trunc && done + p.n_ticks == p_in.n_ticks) ? 1u : 0u;   // the call ends with ONE truncation
    jr_status st = launch_step_once(e, p);
    if (st != JR_OK) return st;
    done += p.n_ticks;
    p.now += (uint64_t)p.n_ticks * p.dt;
    p.step_index += p.n_ticks;
    p.cur ^= (int)(p.n_ticks & 1u);
    if (p.proposals) p.proposals += (size_t)p.n_ticks * p.prop_stride;
    p.tok_tick += p.n_ticks;
    p.phases = PH_RESET_OUT | PH_DRAIN | (p_in.phases & PH_PROPOSE) | PH_TICK;
  }
  return JR_OK;
}

template <int R>
static void launch_sym_r(jr_engine* e, const StepParams& p) {
  if constexpr (R >= 2) {
    // the entry checks, then the fold that consumes their records: nothing may run between the two
    JR_LAUNCH_SMEM(sym_check_kernel<R>, e->d.Gp / 32, 32 * R, sym_check_smem_words(R) * sizeof(uint32_t), e->stream, e->d, p,
                   e->symrec);
    JR_LAUNCH_SMEM(sym2_kernel<R>, (e->d.Gp + SYM2_GROUPS - 1) / SYM2_GROUPS, 2 * SYM2_GROUPS,
                   (size_t)SYM2_UNITS * SYM2_GROUPS * sizeof(uint4), e->stream, e->d, p, e->symdone, e->symblk, e->symrec);
  }
}

// May this launch be offered to the symmetric-group fold?  (Whether a GROUP takes it is sym_check_kernel's decision.)
static bool fold_eligible(const jr_engine* e, const StepParams& p) {
  const Dev& d = e->d;
  const uint32_t whole = PH_RESET_OUT | PH_DRAIN | PH_TICK;
  if (e->no_fold || (d.flags & (JR_F_STREAM_DIGEST | JR_F_SLED_COMMIT_KEY_STRICT | JR_F_NO_SYMMETRIC_FOLD))) return false;
  if (d.R < 2 || d.U < d.R + 7 || d.resident != 0xffu || p.dt == 0) return false;
  if ((p.phases & ~(uint32_t)PH_PROPOSE) != whole || p.n_ticks < 2) return false;
  if (p.proposals && p.prop_stride != d.G) return false;
  return true;   // (tok_runs: always per-tick)
}

static jr_status launch_step_once(jr_engine* e, const StepParams& p_in) {
  const uint32_t n_blocks = e->d.Gp / GROUPS_PER_CTA;
  const size_t smem = step_smem_bytes(e->d);
  StepParams p = p_in;
  p.epoch = (uint32_t)(e->launches_total + 1) * 8u;
  if (fold_eligible(e, p)) {
    DISPATCH_R(e->cfg.n_replicas, (launch_sym_r<RR>(e, p)));
    CK(cudaGetLastError());
    p.symdone = e->symdone;
    p.symblk = e->symblk;
    e->launches_folded += 1;
  }
  e->last_launch_folded = p.symdone != nullptr;
  p.n_parts = choose_parts(e, p, n_blocks);
  // When the fold has been taking every group (no launch of the last two left one behind -- a hint the kernel stores in
  // mapped host memory), step_kernel's CTAs only look at symblk and return: do not cut them in parts, which would cost
  // each of them a ticket and two barriers first.  A wrong guess costs balance in that one launch, nothing else.
  if (p.symdone && e->h_unfolded && (*e->h_unfolded == 0 || p.epoch - *e->h_unfolded > 2u * 8u) && !e->force_parts)
    p.n_parts = 1;
  p.part_ticks = (p.n_ticks + p.n_parts - 1) / p.n_parts;
  p.n_parts = (p.n_ticks + p.part_ticks - 1) / p.part_ticks;  // no empty trailing part
  p.n_blocks = n_blocks;
  const uint32_t grid = n_blocks * p.n_parts;
  // Variant choice from the (possibly one launch stale) scatter flag: it only affects speed.
  // (the kernel stores its epoch into that mapped host word: no memset, no copy-back in the launch path)
  const bool sorted = e->force_sorted > 0 || (e->force_sorted == 0 && e->h_scatter && *e->h_scatter != 0 && p.epoch - *e->h_scatter <= 2u * 8u);
  p.ticket_base = e->ticket_sum;
  if (p.n_parts > 1) e->ticket_sum += grid;
  DISPATCH_R(e->cfg.n_replicas, (launch_step_r<RR>(e, p, sorted, grid, smem)));
  CK(cudaGetLastError());
  if (p.trunc) {   // sym2_kernel truncated the groups it folded
    JR_LAUNCH(truncate_kernel, (e->d.Gp + 127) / 128, 128, e->stream, e->d, p.trunc_margin, (const uint8_t*)p.symdone);
    CK(cudaGetLastError());
  }
  e->launches_sorted += sorted ? 1 : 0;
  e->launches_split += p.n_parts > 1 ? 1 : 0;
  e->launches_total += 1;
  return JR_OK;
}

extern "C" {

#ifdef JR_EMU
// Marker of the TEST-ONLY host build (tests/emu): the package loader refuses a library that has it.
int jr_is_emulation(void) { return 1; }
#endif

const char* jr_last_error(void) { return g_err; }

void jr_config_default(jr_config* cfg, uint32_t n_groups, uint32_t n_replicas) {
  if (!cfg) return;
  memset(cfg, 0, sizeof *cfg);
  cfg->abi_version = JR_ABI_VERSION;
  cfg->n_groups = n_groups;
  cfg->n_replicas = n_replicas;
  cfg->election_min_ms = 500;   // mod.rs:318
  cfg->election_max_ms = 1000;  // mod.rs:319
  cfg->heartbeat_ms = 100;      // config.rs:104
  cfg->chain_capacity = 4096;
  cfg->mailbox_units = 64;
  cfg->fsm_units = 64;
}

uint32_t jr_election_timeout(uint64_t seed, uint64_t group, uint32_t node, uint32_t draw, uint32_t mn,
                             uint32_t mx) {
  return election_timeout_draw(seed, group, node, draw, mn, mx);
}

jr_status jr_engine_create(const jr_config* cfg, jr_engine** out) {
  if (!cfg || !out) return JR_E_INVAL;
  // RaftConfig::validate analogue (config.rs:60-84)
  if (cfg->abi_version != JR_ABI_VERSION) { set_err("abi_version mismatch"); return JR_E_INVAL; }
  if (cfg->n_replicas < 1 || cfg->n_replicas > JR_MAX_REPLICAS || cfg->n_groups < 1) { set_err("bad G/R"); return JR_E_INVAL; }
  if (cfg->election_max_ms <= cfg->election_min_ms) { set_err("empty election timeout range"); return JR_E_INVAL; }
  // RaftConfig::validate, config.rs:70-75 (the rules that have a counterpart here)
  if (cfg->heartbeat_ms < 5) { set_err("heartbeat timeout is too low"); return JR_E_INVAL; }
  if (cfg->election_min_ms < 5) { set_err("election timeout is too low"); return JR_E_INVAL; }
  if (cfg->chain_capacity < 2 || cfg->chain_capacity > 0x40000000u) { set_err("chain_capacity out of range"); return JR_E_INVAL; }
  if (cfg->mailbox_units < 8 || cfg->fsm_units < 1) { set_err("mailbox_units >= 8, fsm_units >= 1"); return JR_E_INVAL; }
  if (cfg->fsm_units > (1u << 20) || cfg->fsm_raw_units > (1u << 20) || (cfg->fsm_raw_units && cfg->fsm_raw_units < 32)) {
    set_err("fsm_units <= 2^20, 32 <= fsm_raw_units <= 2^20");
    return JR_E_INVAL;
  }
  if ((cfg->flags & JR_F_CLIENT_RESPONSES) && !(cfg->flags & JR_F_CAPTURE_FSM)) {
    set_err("JR_F_CLIENT_RESPONSES requires JR_F_CAPTURE_FSM");
    return JR_E_INVAL;
  }
  if ((cfg->flags & JR_F_LINK_QUEUES) && !(cfg->flags & JR_F_PEER_LINKS)) {
    set_err("JR_F_LINK_QUEUES requires JR_F_PEER_LINKS");
    return JR_E_INVAL;
  }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    set_err("no CUDA device; this library has no CPU fallback");
    return JR_E_NO_DEVICE;
  }
  if (cfg->device < 0 || cfg->device >= ndev) { set_err("device ordinal %d out of range", cfg->device); return JR_E_INVAL; }
  CK(cudaSetDevice(cfg->device));
  jr_engine* e = new (std::nothrow) jr_engine();
  if (!e) return JR_E_NOMEM;
  e->cfg = *cfg;
  Dev& d = e->d;
  memset(&d, 0, sizeof d);
  d.G = cfg->n_groups;
  d.Gp = (cfg->n_groups + GROUPS_PER_CTA - 1) / GROUPS_PER_CTA * GROUPS_PER_CTA;
  d.R = cfg->n_replicas;
  d.cap = cfg->chain_capacity;
  d.capm = 1;
  while (d.capm < d.cap) d.capm <<= 1;   // table rows: the power of two >= cap, so row = id & capm
  d.capm -= 1;
  d.U = cfg->mailbox_units;
  d.F = cfg->fsm_units;
  d.Fr = cfg->fsm_raw_units ? cfg->fsm_raw_units : 192u;
  d.flags = cfg->flags;
  d.emin = cfg->election_min_ms;
  d.emax = cfg->election_max_ms;
  d.hb = cfg->heartbeat_ms;
  d.seed = cfg->seed;
  d.goff = cfg->group_offset;
  // shared-memory staging: Us mailbox units per replica per buffer, W table-cache entries
  d.Us = std::min<uint32_t>(cfg->mailbox_units, 6u);
  d.W = 4;
  d.use_index = getenv("JR_NO_INDEX") ? 0u : 1u;
  d.resident = cfg->resident_mask ? cfg->resident_mask : 0xffu;
  if (const char* ev = getenv("JR_SMEM_UNITS")) d.Us = std::min<uint32_t>(cfg->mailbox_units, (uint32_t)atoi(ev));
  if (const char* ev = getenv("JR_TABLE_CACHE")) { uint32_t w = (uint32_t)atoi(ev); d.W = (w & (w - 1)) ? 8 : w; }
  const size_t plane = (size_t)d.R * d.Gp;
  jr_status st = JR_OK;
#define A(ptr, n) if (st == JR_OK) st = dalloc(e, &(ptr), (n))
  A(d.p0, plane); A(d.p1, plane); A(d.p2, plane); A(d.p3, plane);
  A(d.pr, plane * ((d.R + 3) / 4));
  A(d.mk, plane);
  A(d.qt, plane * JR_CLIENT_QUEUE_CAP);
  A(d.dg, plane); A(d.cn, plane);
  A(d.cnext, plane * ((size_t)d.capm + 1));
  A(d.ctok, plane * ((size_t)d.capm + 1));
  A(d.ob[0], plane * (size_t)d.U); A(d.ob[1], plane * (size_t)d.U);
  A(d.oc[0], plane); A(d.oc[1], plane);
  A(d.fs, plane * (size_t)((d.flags & JR_F_CAPTURE_FSM) ? 2 * (size_t)d.F : 1));
  A(d.fc, plane);
  A(d.fq, plane);
  A(d.fr, plane * (size_t)((d.flags & JR_F_CAPTURE_FSM) ? d.Fr : 1));
  A(d.tb, d.Gp);
  A(e->symdone, d.Gp);
  A(e->symblk, d.Gp / GROUPS_PER_CTA);
  A(e->symrec, (size_t)sym_record_words(d.R) * d.Gp);
  if (d.flags & JR_F_PEER_LINKS) A(d.links, d.Gp);   // (padded groups too: step_kernel's lanes read their row)
  if (d.flags & JR_F_LINK_QUEUES) {                   // (R = 1: one slot, never used, so that every pointer is set)
    const size_t slots = std::max<uint32_t>(d.R - 1, 1u);
    A(d.lq, (size_t)LQ_UNITS * slots * plane);
    A(d.lqc, slots * plane);
    A(d.lqm, d.Gp);
  }
  if (d.flags & JR_F_CAPTURE_FSM) {
    const size_t reps = (size_t)cfg->n_groups * cfg->n_replicas;   // default: 2 per replica, but never less than a small engine's whole FIFO space
    const size_t want = cfg->fsm_host_records ? cfg->fsm_host_records
                                              : std::max(3 * reps + 1024, std::min<size_t>(reps * cfg->fsm_units, 1u << 16));
    e->fsm_cap = (uint32_t)std::min<size_t>(want, 0x7fffffffu);
    if (d.flags & JR_F_CLIENT_RESPONSES) {
      e->resp_cap = e->fsm_cap;
      // PN runs, the run counts and the restart marks in one allocation: one checkpoint segment
      uint4* pn = nullptr;
      A(pn, pn_units(plane));
      e->rp.pn = pn;
      if (pn) {
        e->rp.pnc = reinterpret_cast<uint32_t*>(pn + 2 * (size_t)JR_NOTIFY_RUNS * plane);
        e->rp.rm = pn + 2 * (size_t)JR_NOTIFY_RUNS * plane + (plane + 3) / 4;
      }
      A(e->rp.rs, plane * 2 * (size_t)d.F);
      A(e->rp.rc, plane);
      A(e->rp.rd, plane);
    }
    const size_t n_hdr = e->resp_cap ? 2 : 1;
    A(e->fsm_part, 3 * plane);   // (sized for one-thread CTAs, which is what the CPU emulation launches)
    for (int i = 0; i < jr_engine::NSLOT; ++i) {
      A(e->fsm_stage[i], 2 * ((size_t)e->fsm_cap + e->resp_cap));
      A(e->fsm_stage_hdr[i], n_hdr);
    }
  }
  A(e->scratch, 8);
  A(d.scatter, 2);
  A(d.done, d.Gp / GROUPS_PER_CTA);
#ifdef JR_PROFILE
  A(d.prof, 3 * 16 * 2);
#endif
#ifdef JR_SYM_ABORT_LOG
  A(d.sab, 2 * (size_t)d.Gp);
#endif
  for (int i = 0; i < jr_engine::NBUF; ++i) { A(e->prop[i], d.G); A(e->leaders[i], d.G); }
  A(e->route, d.G);
#undef A
  if (st != JR_OK) { jr_engine_destroy(e); return st; }
  if (cudaStreamCreateWithFlags(&e->own_stream, cudaStreamNonBlocking) != cudaSuccess) {
    set_err("cudaStreamCreate failed");
    jr_engine_destroy(e);
    return JR_E_CUDA;
  }
  e->stream = e->own_stream;
  {
    bool ok = cudaStreamCreateWithFlags(&e->h2d, cudaStreamNonBlocking) == cudaSuccess &&
              cudaStreamCreateWithFlags(&e->d2h, cudaStreamNonBlocking) == cudaSuccess;
    for (int i = 0; ok && i < jr_engine::NBUF; ++i)
      ok = cudaEventCreateWithFlags(&e->prop_ready[i], cudaEventDisableTiming) == cudaSuccess &&
           cudaEventCreateWithFlags(&e->prop_free[i], cudaEventDisableTiming) == cudaSuccess &&
           cudaEventCreateWithFlags(&e->tab_ready[i], cudaEventDisableTiming) == cudaSuccess &&
           cudaEventCreateWithFlags(&e->tab_free[i], cudaEventDisableTiming) == cudaSuccess &&
           cudaEventCreateWithFlags(&e->batch_ready[i], cudaEventDisableTiming) == cudaSuccess &&
           cudaEventCreateWithFlags(&e->batch_free[i], cudaEventDisableTiming) == cudaSuccess;
    for (int i = 0; ok && i < jr_engine::NSLOT; ++i)
      ok = cudaEventCreateWithFlags(&e->fsm_packed[i], cudaEventDisableTiming) == cudaSuccess &&
           cudaEventCreateWithFlags(&e->fsm_landed[i], cudaEventDisableTiming) == cudaSuccess;
    for (int i = 0; ok && e->fsm_cap && i < jr_engine::NSLOT; ++i)   // the drain's landing buffers: pinned, device-visible
      ok = cudaHostAlloc((void**)&e->fsm_host[i], ((size_t)e->fsm_cap + e->resp_cap) * sizeof(jr_fsm_record), cudaHostAllocMapped) == cudaSuccess &&
           cudaHostAlloc((void**)&e->fsm_host_hdr[i], (e->resp_cap ? 2 : 1) * sizeof(FsmHeader), cudaHostAllocMapped) == cudaSuccess;
    if (!ok) {
      set_err("copy streams / events could not be created");
      jr_engine_destroy(e);
      return JR_E_CUDA;
    }
  }
  {
    const int smem = (int)step_smem_bytes(d);
    cudaError_t aerr = cudaSuccess;
    DISPATCH_R(d.R, (aerr = step_smem_attr_r<RR>(smem, d.lq != nullptr)));
    if (aerr == cudaSuccess) aerr = cudaHostAlloc((void**)&e->h_scatter, sizeof(uint32_t), cudaHostAllocMapped);
    if (aerr == cudaSuccess) *e->h_scatter = 0;
    if (aerr == cudaSuccess) aerr = cudaHostGetDevicePointer((void**)&e->d.hscat, (void*)e->h_scatter, 0);
    if (aerr == cudaSuccess) aerr = cudaHostAlloc((void**)&e->h_unfolded, sizeof(uint32_t), cudaHostAllocMapped);
    if (aerr == cudaSuccess) *e->h_unfolded = 0;
    if (aerr == cudaSuccess) aerr = cudaHostGetDevicePointer((void**)&e->d.hunf, (void*)e->h_unfolded, 0);
    if (const char* ev = getenv("JR_NO_FOLD")) e->no_fold = atoi(ev);
    if (const char* ev = getenv("JR_PARTS")) e->force_parts = (uint32_t)std::min(std::max(atoi(ev), 0), 8);
#ifndef JR_EMU
    if (aerr == cudaSuccess) {
      int per_sm = 0, sms = 0;
      DISPATCH_R(d.R, (aerr = step_occupancy_r<RR>(&per_sm, smem)));
      if (aerr == cudaSuccess) aerr = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, cfg->device);
      e->slots = (uint32_t)(per_sm * sms);
      e->sms = (uint32_t)sms;
    }
#endif
    if (const char* ev = getenv("JR_STEP_VARIANT")) e->force_sorted = !strcmp(ev, "sorted") ? 1 : (!strcmp(ev, "plain") ? -1 : 0);
    if (aerr != cudaSuccess) {
      set_err("step kernel needs %d bytes of shared memory: %s", smem, cudaGetErrorString(aerr));
      jr_engine_destroy(e);
      return JR_E_CUDA;
    }
  }
  if (jr_engine_reset(e) != JR_OK) {
    jr_engine_destroy(e);
    return JR_E_CUDA;
  }
  *out = e;
  return JR_OK;
}

#ifdef JR_PROFILE
// Profiling builds only (not part of the ABI): read and clear the phase counters.
jr_status jr_profile_read(jr_engine* e, unsigned long long* out96) {
  if (!e || !out96) return JR_E_INVAL;
  CK(cudaStreamSynchronize(e->stream));
  CK(cudaMemcpyAsync(out96, e->d.prof, 96 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaMemsetAsync(e->d.prof, 0, 96 * sizeof(unsigned long long), e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return JR_OK;
}
#endif

#ifdef JR_SYM_ABORT_LOG
// Abort-log builds only (tests/emu; not part of the ABI): read and clear the fold's abort records, out[lane * G + g] =
// the first abort site | tick << 8 of group g's lane since the last read, 0 = none (sym_fold.cuh, SA_*).
jr_status jr_sym_abort_read(jr_engine* e, uint32_t* out, size_t n) {
  if (!e || !out || n < 2 * (size_t)e->d.G) return JR_E_INVAL;
  CK(cudaStreamSynchronize(e->stream));
  for (int lane = 0; lane < 2; ++lane)
    CK(cudaMemcpyAsync(out + (size_t)lane * e->d.G, e->d.sab + (size_t)lane * e->d.Gp, e->d.G * sizeof(uint32_t),
                       cudaMemcpyDeviceToHost, e->stream));
  CK(cudaMemsetAsync(e->d.sab, 0, 2 * (size_t)e->d.Gp * sizeof(uint32_t), e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return JR_OK;
}
#endif

jr_status jr_engine_reset(jr_engine* e) {
  if (!e) return JR_E_INVAL;
  CK(cudaSetDevice(e->cfg.device));
  const Dev& d = e->d;
  const size_t plane = (size_t)d.R * d.Gp;
  // block tables start empty (all keys absent); pr / qt zero
  CK(cudaMemsetAsync(d.cnext, 0xFF, plane * ((size_t)d.capm + 1) * sizeof(uint32_t), e->stream));
  CK(cudaMemsetAsync(d.pr, 0, plane * ((d.R + 3) / 4) * sizeof(uint4), e->stream));
  CK(cudaMemsetAsync(d.qt, 0, plane * JR_CLIENT_QUEUE_CAP * sizeof(uint4), e->stream));
  CK(cudaMemsetAsync(e->route, 0, (size_t)d.G * sizeof(uint32_t), e->stream));  // no leader announced yet
  CK(cudaMemsetAsync(d.done, 0, (size_t)(d.Gp / GROUPS_PER_CTA) * sizeof(uint32_t), e->stream));
  CK(cudaMemsetAsync(d.scatter, 0, 2 * sizeof(uint32_t), e->stream));   // [1] = the ticket counter: from here on only launches move it,
  e->ticket_sum = 0;                                                     //       and each one is told where it stands (ticket_base)
  if (e->rp.pnc)   // every fsm::Driver map empty, no restart pending
    CK(cudaMemsetAsync(e->rp.pnc, 0, ((plane + 3) / 4 + plane) * sizeof(uint4), e->stream));
  e->resp_b = -1;
  if (d.links) CK(cudaMemsetAsync(d.links, 0, (size_t)d.Gp * sizeof(unsigned long long), e->stream));   // fully connected
  if (d.lq) {   // every link queue empty (the units too: a checkpoint's bytes depend only on what the engine did)
    const size_t slots = std::max<uint32_t>(d.R - 1, 1u);
    CK(cudaMemsetAsync(d.lq, 0, (size_t)LQ_UNITS * slots * plane * sizeof(uint4), e->stream));
    CK(cudaMemsetAsync(d.lqc, 0, slots * plane * sizeof(uint32_t), e->stream));
    CK(cudaMemsetAsync(d.lqm, 0, (size_t)d.Gp * sizeof(unsigned long long), e->stream));
  }
  JR_LAUNCH(init_kernel, (unsigned)((plane + 255) / 256), 256, e->stream, d);
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(e->stream));
  e->cur = 0;
  e->step_index = 0;
  // (h_scatter keeps its last value: advisory only, and a reset is usually followed by the same workload)
#ifdef JR_PROFILE
  CK(cudaMemsetAsync(e->d.prof, 0, 96 * sizeof(unsigned long long), e->stream));
#endif
#ifdef JR_SYM_ABORT_LOG
  CK(cudaMemsetAsync(e->d.sab, 0, 2 * (size_t)d.Gp * sizeof(uint32_t), e->stream));
#endif
  return JR_OK;
}

void jr_engine_destroy(jr_engine* e) {
  if (!e) return;
  if (getenv("JR_DEBUG_VARIANT"))
    fprintf(stderr, "[jr] engine %p: %llu step launches, %llu role-sorted, %llu split, %llu offered to the fold; %u CTA slots\n",
            (void*)e, (unsigned long long)e->launches_total, (unsigned long long)e->launches_sorted,
            (unsigned long long)e->launches_split, (unsigned long long)e->launches_folded, e->slots);
  cudaSetDevice(e->cfg.device);
  if (e->stream) cudaStreamSynchronize(e->stream);
  for (void* p : e->allocs) cudaFree(p);
  if (e->inj_msgs) cudaFree(e->inj_msgs);
  if (e->inj_targets) cudaFree(e->inj_targets);
  if (e->many_buf) cudaFree(e->many_buf);
  if (e->verify_buf) cudaFree(e->verify_buf);
  if (e->move_buf) cudaFree(e->move_buf);
  if (e->move_img) cudaFree(e->move_img);
  if (e->h2d) { cudaStreamSynchronize(e->h2d); cudaStreamDestroy(e->h2d); }
  if (e->d2h) { cudaStreamSynchronize(e->d2h); cudaStreamDestroy(e->d2h); }
  for (int i = 0; i < jr_engine::NBUF; ++i) {
    if (e->prop_ready[i]) cudaEventDestroy(e->prop_ready[i]);
    if (e->prop_free[i]) cudaEventDestroy(e->prop_free[i]);
    if (e->tab_ready[i]) cudaEventDestroy(e->tab_ready[i]);
    if (e->tab_free[i]) cudaEventDestroy(e->tab_free[i]);
    if (e->batch_ready[i]) cudaEventDestroy(e->batch_ready[i]);
    if (e->batch_free[i]) cudaEventDestroy(e->batch_free[i]);
    if (e->batch[i]) cudaFree(e->batch[i]);
    if (e->tokbuf[i]) cudaFree(e->tokbuf[i]);
  }
  for (int i = 0; i < jr_engine::NSLOT; ++i) {
    if (e->fsm_packed[i]) cudaEventDestroy(e->fsm_packed[i]);
    if (e->fsm_landed[i]) cudaEventDestroy(e->fsm_landed[i]);
    if (e->fsm_host[i]) cudaFreeHost(e->fsm_host[i]);
    if (e->fsm_host_hdr[i]) cudaFreeHost(e->fsm_host_hdr[i]);
  }
  if (e->h_scatter) cudaFreeHost((void*)e->h_scatter);
  if (e->h_unfolded) cudaFreeHost((void*)e->h_unfolded);
  if (e->own_stream) cudaStreamDestroy(e->own_stream);
  delete e;
}

jr_status jr_engine_set_stream(jr_engine* e, void* s) {
  if (!e) return JR_E_INVAL;
  CK(cudaStreamSynchronize(e->stream));
  e->stream = s ? (cudaStream_t)s : e->own_stream;
  return JR_OK;
}

jr_status jr_engine_sync(jr_engine* e) {
  if (!e) return JR_E_INVAL;
  CK(cudaStreamSynchronize(e->h2d));
  CK(cudaStreamSynchronize(e->stream));
  CK(cudaStreamSynchronize(e->d2h));
  return JR_OK;
}

// ---- capture: decode raw mailboxes / FIFOs on the host --------------------------------

static void decode_unit(const uint4& h, uint32_t group, uint32_t sender, const uint4* blocks, size_t stride,
                        std::vector<jr_msg>& out) {
  const uint32_t kind = h.x & 15u, flag = (h.x >> 4) & 1u, aux = (h.x >> 8) & 255u, to = h.x >> 16;
  jr_msg m;
  memset(&m, 0, sizeof m);
  m.group = group;
  m.from_kind = JR_ADDR_PEER;
  m.from_id = sender;
  m.to_kind = to == TO_PEERS ? JR_ADDR_PEERS : (to == TO_CLIENT ? JR_ADDR_CLIENT : JR_ADDR_PEER);
  m.to_id = m.to_kind == JR_ADDR_PEER ? to : 0;
  m.kind = (uint8_t)kind;
  const uint64_t t = (uint64_t)h.y | ((uint64_t)h.z << 32);
  uint32_t copies = 1;
  switch (kind) {
    case JR_CMD_VOTE_REQUEST: m.term = t; m.node_id = sender; m.last_term = t; m.block = h.w; copies = aux; break;
    case JR_CMD_VOTE_RESPONSE: m.term = t; m.node_id = sender; m.flag = flag; break;
    case JR_CMD_APPEND_ENTRIES:
      m.term = t; m.node_id = sender; m.n_blocks = (uint8_t)aux;
      for (uint32_t k = 0; k < aux && k < JR_MAX_AE_BLOCKS; ++k) {
        const uint4& b = blocks[(size_t)k * stride];
        m.blocks[k] = jr_block{b.x, b.y, (uint64_t)b.z | ((uint64_t)b.w << 32)};
      }
      break;
    case JR_CMD_APPEND_RESPONSE: m.node_id = sender; m.term = t; m.block = h.w; m.flag = flag; break;
    case JR_CMD_HEARTBEAT: m.term = t; m.block = h.w; m.node_id = sender; break;
    case JR_CMD_HEARTBEAT_RESPONSE: m.block = h.w; m.flag = flag; break;
    case JR_CMD_CLIENT_REQUEST: m.token = t; m.client_kind = (uint8_t)(h.w >> 16); m.client_id = h.w & 0xffffu; break;
    case JR_CMD_CLIENT_RESPONSE: m.token = t; break;
    default: break;
  }
  for (uint32_t k = 0; k < copies; ++k) out.push_back(m);
}

static jr_status device_max(jr_engine* e, const uint32_t* v, size_t n, uint32_t* out) {
  uint32_t* s = reinterpret_cast<uint32_t*>(e->scratch);
  CK(cudaMemsetAsync(s, 0, sizeof(uint32_t), e->stream));
  JR_LAUNCH(max_u32_kernel, 64, CTA_THREADS, e->stream, v, n, s);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out, s, sizeof(uint32_t), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return JR_OK;
}

static jr_status capture_messages(jr_engine* e, int buf, std::vector<jr_msg>& out) {
  const Dev& d = e->d;
  const size_t plane = (size_t)d.R * d.Gp;
  uint32_t mx = 0;
  jr_status st = device_max(e, d.oc[buf], plane, &mx);
  if (st != JR_OK) return st;
  std::vector<uint32_t> cnt(plane);
  CK(cudaMemcpyAsync(cnt.data(), d.oc[buf], plane * sizeof(uint32_t), cudaMemcpyDeviceToHost, e->stream));
  std::vector<uint4> units((size_t)mx * plane);
  if (mx) CK(cudaMemcpyAsync(units.data(), d.ob[buf], units.size() * sizeof(uint4), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  for (uint32_t g = 0; g < d.G; ++g)
    for (uint32_t r = 0; r < d.R; ++r) {
      const size_t i = (size_t)r * d.Gp + g;
      for (uint32_t u = 0; u < cnt[i];) {
        const uint4& h = units[(size_t)u * plane + i];
        const uint32_t kind = h.x & 15u, aux = (h.x >> 8) & 255u;
        const bool ae = kind == JR_CMD_APPEND_ENTRIES, ref = ae && ((h.x >> 4) & 1u);
        const uint32_t span = 1 + ((ae && !ref) ? aux : 0u);
        const uint32_t first = ref ? h.w : u + 1;  // block run: inline, or shared with an earlier AppendEntries
        decode_unit(h, g, r + 1, (ae && aux) ? &units[(size_t)first * plane + i] : nullptr, plane, out);
        u += span;
      }
    }
  return JR_OK;
}

// ---- Instruction-stream drain -----------------------------------------------------------------

static jr_status fsm_records_enqueue(jr_engine* e) {
  const Dev& d = e->d;
  if (!(d.flags & JR_F_CAPTURE_FSM)) { set_err("engine created without JR_F_CAPTURE_FSM"); return JR_E_INVAL; }
  size_t last_records, last_resp;
  {
    std::lock_guard<std::mutex> l(e->qmu);
    if (e->fsm_npending == jr_engine::NBUF) { set_err("%d batches outstanding: call jr_fsm_records_wait first", jr_engine::NBUF); return JR_E_INVAL; }
    last_records = e->fsm_last_records;
    last_resp = e->resp_last;
  }
  const int b = e->fsm_i;
  e->fsm_i = (b + 1) % jr_engine::NSLOT;
  const size_t plane = (size_t)d.R * d.Gp;
  if (e->fsm_used[b]) CK(cudaStreamWaitEvent(e->stream, e->fsm_landed[b], 0));  // stage[b] has left the device
  const uint32_t T = CTA_THREADS, Ts = SCAN_THREADS;
  const uint32_t n_ctas = (uint32_t)((plane + T - 1) / T);
  JR_LAUNCH(fsm_count_kernel, n_ctas, T, e->stream, d, d.fc, nullptr, e->fsm_part, n_ctas);
  CK(cudaGetLastError());
  JR_LAUNCH(fsm_scan_kernel, 1, Ts, e->stream, e->fsm_part, n_ctas, e->fsm_stage_hdr[b], e->fsm_cap, false);
  CK(cudaGetLastError());
  if (e->resp_cap) {   // reads the FIFOs before the pack empties them
    JR_LAUNCH(fsm_respond_kernel, n_ctas, T, e->stream, d, e->rp, e->fsm_stage_hdr[b], e->fsm_cap);
    CK(cudaGetLastError());
  }
  JR_LAUNCH(fsm_pack_kernel, n_ctas, T, e->stream, d, d.fs, d.fc, e->fsm_part, e->fsm_stage_hdr[b], e->fsm_stage[b], e->fsm_cap,
            false);
  CK(cudaGetLastError());
  uint4* const resp_stage = e->fsm_stage[b] + 2 * (size_t)e->fsm_cap;
  if (e->resp_cap) {
    JR_LAUNCH(fsm_count_kernel, n_ctas, T, e->stream, d, e->rp.rc, e->rp.rd, e->fsm_part, n_ctas);
    CK(cudaGetLastError());
    JR_LAUNCH(fsm_scan_kernel, 1, Ts, e->stream, e->fsm_part, n_ctas, e->fsm_stage_hdr[b] + 1, e->resp_cap, true);
    CK(cudaGetLastError());
    JR_LAUNCH(fsm_pack_kernel, n_ctas, T, e->stream, d, e->rp.rs, e->rp.rc, e->fsm_part, e->fsm_stage_hdr[b] + 1, resp_stage,
              e->resp_cap, true);
    CK(cudaGetLastError());
  }
  CK(cudaEventRecord(e->fsm_packed[b], e->stream));
  CK(cudaStreamWaitEvent(e->d2h, e->fsm_packed[b], 0));
  // Copy engine, speculatively: the batch size is only known on the device, so copy as many records as the previous
  // batch held plus a margin; fsm_records_take fetches the rest in the (rare) case the batch turned out larger.
  // (A copy by the SMs would store to host memory with load/store units the next step's kernel needs: every SM runs
  // equal CTAs, so the slowest SM sets its duration.  A DMA copy takes nothing from the SMs.)
  const size_t guess = std::min<size_t>(e->fsm_cap, std::max<size_t>(last_records + last_records / 8 + 1024, 16384));
  if (guess) CK(cudaMemcpyAsync(e->fsm_host[b], e->fsm_stage[b], guess * sizeof(jr_fsm_record), cudaMemcpyDeviceToHost, e->d2h));
  CK(cudaMemcpyAsync(e->fsm_host_hdr[b], e->fsm_stage_hdr[b], sizeof(FsmHeader), cudaMemcpyDeviceToHost, e->d2h));
  e->fsm_copied[b] = guess;
  if (e->resp_cap) {   // the same scheme for the responses
    const size_t rg = std::min<size_t>(e->resp_cap, std::max<size_t>(last_resp + last_resp / 8 + 1024, 16384));
    CK(cudaMemcpyAsync(e->fsm_host[b] + 2 * (size_t)e->fsm_cap, resp_stage, rg * sizeof(jr_fsm_record), cudaMemcpyDeviceToHost, e->d2h));
    CK(cudaMemcpyAsync(e->fsm_host_hdr[b] + 1, e->fsm_stage_hdr[b] + 1, sizeof(FsmHeader), cudaMemcpyDeviceToHost, e->d2h));
    e->resp_copied[b] = rg;
  }
  CK(cudaEventRecord(e->fsm_landed[b], e->d2h));
  e->fsm_used[b] = true;
  std::lock_guard<std::mutex> l(e->qmu);
  e->fsm_pending[e->fsm_npending++] = b;
  return JR_OK;
}

static jr_status fsm_records_take(jr_engine* e, const jr_fsm_record** recs, jr_fsm_batch* batch) {
  int b;
  {
    std::lock_guard<std::mutex> l(e->qmu);
    if (e->fsm_npending == 0) { set_err("no batch outstanding"); return JR_E_INVAL; }
    b = e->fsm_pending[0];
    for (int k = 0; k + 1 < jr_engine::NBUF; ++k) e->fsm_pending[k] = e->fsm_pending[k + 1];
    --e->fsm_npending;
  }
  CK(cudaEventSynchronize(e->fsm_landed[b]));
  const FsmHeader& h = *e->fsm_host_hdr[b];
  if (h.n_records > e->fsm_copied[b]) {   // the speculative copy was short: fetch the tail now (stage[b] is still intact)
    const size_t have = e->fsm_copied[b];
    CK(cudaMemcpyAsync(reinterpret_cast<jr_fsm_record*>(e->fsm_host[b]) + have, reinterpret_cast<const jr_fsm_record*>(e->fsm_stage[b]) + have,
                       ((size_t)h.n_records - have) * sizeof(jr_fsm_record), cudaMemcpyDeviceToHost, e->d2h));
    CK(cudaEventRecord(e->fsm_landed[b], e->d2h));
    CK(cudaEventSynchronize(e->fsm_landed[b]));
    e->fsm_copied[b] = h.n_records;
  }
  size_t n_resp = 0;
  if (e->resp_cap) {
    const FsmHeader& hr = e->fsm_host_hdr[b][1];
    n_resp = hr.n_records;
    if (hr.n_records > e->resp_copied[b]) {
      const size_t have = e->resp_copied[b];
      jr_fsm_record* dst = reinterpret_cast<jr_fsm_record*>(e->fsm_host[b] + 2 * (size_t)e->fsm_cap);
      const jr_fsm_record* src = reinterpret_cast<const jr_fsm_record*>(e->fsm_stage[b] + 2 * (size_t)e->fsm_cap);
      CK(cudaMemcpyAsync(dst + have, src + have, ((size_t)hr.n_records - have) * sizeof(jr_fsm_record), cudaMemcpyDeviceToHost, e->d2h));
      CK(cudaEventRecord(e->fsm_landed[b], e->d2h));
      CK(cudaEventSynchronize(e->fsm_landed[b]));
      e->resp_copied[b] = hr.n_records;
    }
  }
  {
    std::lock_guard<std::mutex> l(e->qmu);
    e->fsm_last_records = h.n_records;
    if (e->resp_cap) { e->resp_last = n_resp; e->resp_b = b; }
  }
  if (recs) *recs = reinterpret_cast<const jr_fsm_record*>(e->fsm_host[b]);
  if (batch) {
    memset(batch, 0, sizeof *batch);
    batch->n_records = h.n_records;
    batch->n_dropped = h.n_dropped;
    batch->n_instructions = h.n_instructions;
    for (uint32_t r = 0; r <= JR_MAX_REPLICAS; ++r) batch->node_offset[r] = r <= e->d.R ? h.node_offset[r] : h.node_offset[e->d.R];
  }
  if (h.n_dropped) {
    set_err("%llu Instruction records were dropped (raise fsm_units / fsm_host_records, or drain more often)",
            (unsigned long long)h.n_dropped);
    return JR_E_CAPACITY;
  }
  return JR_OK;
}

// Synchronous drain into expanded Instructions (jr_step capture, jr_drain_fsm).
static jr_status capture_fsm(jr_engine* e, std::vector<jr_fsm_instr>& out) {
  const Dev& d = e->d;
  if (!(d.flags & JR_F_CAPTURE_FSM)) return JR_OK;
  if (e->fsm_npending) { set_err("jr_fsm_records_async batches are outstanding"); return JR_E_INVAL; }
  jr_status st = fsm_records_enqueue(e);
  if (st != JR_OK) return st;
  const jr_fsm_record* recs = nullptr;
  jr_fsm_batch batch;
  const jr_status took = fsm_records_take(e, &recs, &batch);
  if (took != JR_OK) return took;   // JR_E_CAPACITY: records are missing, so what is left cannot be expanded faithfully
  size_t n = 0;
  st = jr_fsm_expand(recs, batch.n_records, d.G, d.R, nullptr, 0, &n);
  if (st != JR_OK && st != JR_E_CAPACITY) return st;
  out.resize(n);
  if (n && (st = jr_fsm_expand(recs, batch.n_records, d.G, d.R, out.data(), n, &n)) != JR_OK) return st;
  return took;
}

// ---- jr_step ------------------------------------------------------------------------------

jr_status jr_step(jr_engine* e, jr_step_args* a) {
  if (!e || !a) return JR_E_INVAL;
  CK(cudaSetDevice(e->cfg.device));
  const Dev& d = e->d;
  const uint32_t R = d.R, G = d.G;
  if (a->n_synth > 8) { set_err("n_synth <= 8"); return JR_E_INVAL; }
  if ((a->out_msgs && !(d.flags & JR_F_CAPTURE_MESSAGES)) || (a->out_fsm && !(d.flags & JR_F_CAPTURE_FSM))) {
    set_err("output buffer given but capture flag not set at create");
    return JR_E_INVAL;
  }
  // ---- validate + bucket injected commands by target, stable
  std::vector<jr_msg> sorted;
  std::vector<uint4> targets;
  if (a->n_inject) {
    if (!a->inject) return JR_E_INVAL;
    std::vector<uint32_t> order(a->n_inject);
    for (size_t i = 0; i < a->n_inject; ++i) {
      const jr_msg& m = a->inject[i];
      if (m.group >= G || m.to_kind != JR_ADDR_PEER) { set_err("inject[%zu]: bad group / to_kind", i); return JR_E_INVAL; }
      if (m.to_id < 1 || m.to_id > R) return JR_E_UNKNOWN_NODE;
      if (m.node_id > JR_MAX_NODE_ID || m.from_id > JR_MAX_NODE_ID || m.client_id > JR_MAX_NODE_ID) return JR_E_INVAL;
      if (m.kind == JR_CMD_VOTE_RESPONSE && (m.node_id < 1 || m.node_id > 32)) return JR_E_UNKNOWN_NODE;
      if (m.n_blocks > JR_MAX_AE_BLOCKS) return JR_E_INVAL;
      if (m.block >= 0xffffffffull) { set_err("inject[%zu]: block id >= 2^32-1 (D4)", i); return JR_E_INVAL; }
      for (unsigned k = 0; k < m.n_blocks; ++k)
        if (m.blocks[k].id >= 0xffffffffull || m.blocks[k].next >= 0xffffffffull) return JR_E_INVAL;
      order[i] = (uint32_t)i;
    }
    std::stable_sort(order.begin(), order.end(), [&](uint32_t x, uint32_t y) {
      const jr_msg &p = a->inject[x], &q = a->inject[y];
      return p.group != q.group ? p.group < q.group : p.to_id < q.to_id;
    });
    sorted.reserve(a->n_inject);
    for (uint32_t idx : order) {
      const jr_msg& m = a->inject[idx];
      if (targets.empty() || targets.back().x != m.group || targets.back().y != m.to_id - 1)
        targets.push_back(make_uint4(m.group, m.to_id - 1, (uint32_t)sorted.size(), 0));
      targets.back().w++;
      sorted.push_back(m);
    }
  }
  if (a->proposals && !(a->flags & JR_STEP_TRUSTED_PROPOSALS))
    for (uint32_t g = 0; g < G; ++g)
      if (a->proposals[g].node > R) return JR_E_UNKNOWN_NODE;

  StepParams p;
  p.now = a->now_ms;
  p.step_index = e->step_index;
  p.n_synth = (a->flags & JR_STEP_SYNTH_PROPOSALS) ? a->n_synth : 0;
  p.cur = e->cur;
  p.n_ticks = 1;
  p.dt = 0;
  p.prop_stride = 0;
  p.proposals = nullptr;
  int staged = -1;
  if (a->proposals) {
    const int b = e->prop_i;
    e->prop_i = (b + 1) % jr_engine::NBUF;
    if (e->prop_used[b]) CK(cudaStreamWaitEvent(e->h2d, e->prop_free[b], 0));  // its last reader is done
    CK(cudaMemcpyAsync(e->prop[b], a->proposals, (size_t)G * sizeof(jr_proposal), cudaMemcpyHostToDevice, e->h2d));
    CK(cudaEventRecord(e->prop_ready[b], e->h2d));
    CK(cudaStreamWaitEvent(e->stream, e->prop_ready[b], 0));
    p.proposals = e->prop[b];
    staged = b;
  }
  if (e->rp.rm) {   // PH_RESET_FSM below drops the undrained Instructions a pending restart mark points into
    const size_t plane = (size_t)R * d.Gp;
    JR_LAUNCH(restart_marks_rebase_kernel, (unsigned)((plane + 255) / 256), 256, e->stream, d, e->rp.rm);
    CK(cudaGetLastError());
  }
  const uint32_t ph_first = PH_RESET_OUT | PH_RESET_FSM | ((a->flags & JR_STEP_DELIVER) ? PH_DRAIN : 0u);
  const uint32_t ph_last = ((p.proposals || p.n_synth) ? PH_PROPOSE : 0u) | ((a->flags & JR_STEP_TICK) ? PH_TICK : 0u);
  jr_status st;
  if (targets.empty()) {
    p.phases = ph_first | ph_last;
    if ((st = launch_step(e, p)) != JR_OK) return st;
  } else {
    if (sorted.size() > e->inj_cap) {
      if (e->inj_msgs) cudaFree(e->inj_msgs);
      if (e->inj_targets) cudaFree(e->inj_targets);
      e->inj_msgs = nullptr; e->inj_targets = nullptr;
      e->inj_cap = std::max<size_t>(sorted.size() * 2, 64);
      CK(cudaMalloc(&e->inj_msgs, e->inj_cap * sizeof(jr_msg)));
      CK(cudaMalloc(&e->inj_targets, e->inj_cap * sizeof(uint4)));
    }
    CK(cudaMemcpyAsync(e->inj_msgs, sorted.data(), sorted.size() * sizeof(jr_msg), cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(e->inj_targets, targets.data(), targets.size() * sizeof(uint4), cudaMemcpyHostToDevice, e->stream));
    p.phases = ph_first;
    if ((st = launch_step(e, p)) != JR_OK) return st;
    const uint32_t nt = (uint32_t)targets.size();
    DISPATCH_R(R, (JR_LAUNCH(inject_kernel<RR>, (nt + 63) / 64, 64, e->stream, e->d, p, e->inj_msgs, e->inj_targets, nt)));
    CK(cudaGetLastError());
    if (ph_last) {
      p.phases = ph_last;
      if ((st = launch_step(e, p)) != JR_OK) return st;
    }
    CK(cudaStreamSynchronize(e->stream));  // `sorted` / `targets` are stack-owned host buffers
  }
  if (staged >= 0) {  // proposals buffer may be refilled once the kernels of this step are done
    CK(cudaEventRecord(e->prop_free[staged], e->stream));
    e->prop_used[staged] = true;
    CK(cudaEventSynchronize(e->prop_ready[staged]));  // a->proposals has been read: the caller may reuse it on return
  }
  const int written = e->cur;
  e->cur ^= 1;
  e->step_index++;

  // ---- capture (synchronises)
  a->n_msgs = 0;
  a->n_fsm = 0;
  bool ovf = false;
  if (a->out_msgs) {
    std::vector<jr_msg> msgs;
    if ((st = capture_messages(e, written, msgs)) != JR_OK) return st;
    a->n_msgs = msgs.size();
    memcpy(a->out_msgs, msgs.data(), std::min(msgs.size(), a->cap_msgs) * sizeof(jr_msg));
    ovf |= msgs.size() > a->cap_msgs;
  }
  if (a->out_fsm) {
    std::vector<jr_fsm_instr> fsm;
    st = capture_fsm(e, fsm);
    if (st != JR_OK && st != JR_E_CAPACITY) return st;
    a->n_fsm = fsm.size();
    memcpy(a->out_fsm, fsm.data(), std::min(fsm.size(), a->cap_fsm) * sizeof(jr_fsm_instr));
    ovf |= fsm.size() > a->cap_fsm || st == JR_E_CAPACITY;
  }
  if (a->flags & JR_STEP_REPORT_FAULTS) {
    uint64_t v[5];
    if ((st = stream_sums(e, v)) != JR_OK) return st;
    a->n_faulted = v[4];
  }
  return ovf ? JR_E_CAPACITY : JR_OK;
}

jr_status jr_run(jr_engine* e, uint64_t now0, uint32_t dt, uint32_t n_steps, uint32_t n_synth) {
  if (!e) return JR_E_INVAL;
  if (n_synth > 8) { set_err("n_synth <= 8"); return JR_E_INVAL; }
  CK(cudaSetDevice(e->cfg.device));
  if (n_steps == 0) return JR_OK;
  StepParams p;
  p.now = now0;
  p.step_index = e->step_index;
  p.n_synth = n_synth;
  p.n_ticks = n_steps;
  p.dt = dt;
  p.cur = e->cur;
  p.proposals = nullptr;
  p.prop_stride = 0;
  p.phases = PH_RESET_OUT | PH_DRAIN | (n_synth ? PH_PROPOSE : 0u) | PH_TICK;   // Instructions accumulate until drained
  p.trunc = e->auto_trunc ? 1u : 0u;
  p.trunc_margin = e->auto_trunc_margin;
  jr_status st = launch_step(e, p);
  if (st != JR_OK) return st;
  e->cur ^= (int)(n_steps & 1u);
  e->step_index += n_steps;
  return JR_OK;
}

// Grow batch[b] to n entries once its last reader is done; returns with the h2d stream fenced on that reader.
static jr_status batch_reserve(jr_engine* e, int b, size_t n) {
  if (e->batch_used[b]) CK(cudaStreamWaitEvent(e->h2d, e->batch_free[b], 0));  // its last reader is done
  if (n > e->batch_cap[b]) {
    if (e->batch_used[b]) CK(cudaEventSynchronize(e->batch_free[b]));
    if (e->batch[b]) cudaFree(e->batch[b]);
    e->batch[b] = nullptr;
    e->batch_cap[b] = 0;
    CK(cudaMalloc(&e->batch[b], n * sizeof(jr_proposal)));
    e->batch_cap[b] = n;
  }
  return JR_OK;
}

// The fused launch over batch[b] (already ordered after whatever filled it on e->stream).
static jr_status batch_launch(jr_engine* e, int b, uint64_t now0, uint32_t dt, uint32_t n_steps) {
  StepParams p;
  p.now = now0;
  p.step_index = e->step_index;
  p.n_synth = 0;
  p.n_ticks = n_steps;
  p.dt = dt;
  p.cur = e->cur;
  p.proposals = e->batch[b];
  p.prop_stride = e->d.G;
  p.phases = PH_RESET_OUT | PH_DRAIN | PH_PROPOSE | PH_TICK;
  p.trunc = e->auto_trunc ? 1u : 0u;
  p.trunc_margin = e->auto_trunc_margin;
  jr_status st = launch_step(e, p);
  if (st != JR_OK) return st;
  CK(cudaEventRecord(e->batch_free[b], e->stream));
  e->batch_used[b] = true;
  e->cur ^= (int)(n_steps & 1u);
  e->step_index += n_steps;
  return JR_OK;
}

jr_status jr_run_proposals(jr_engine* e, uint64_t now0, uint32_t dt, uint32_t n_steps, const jr_proposal* proposals,
                           uint32_t flags) {
  if (!e || !proposals) return JR_E_INVAL;
  if (n_steps == 0) return JR_OK;
  CK(cudaSetDevice(e->cfg.device));
  const uint32_t G = e->d.G, R = e->d.R;
  const size_t n = (size_t)n_steps * G;
  if (!(flags & JR_STEP_TRUSTED_PROPOSALS))
    for (size_t i = 0; i < n; ++i)
      if (proposals[i].node > R) return JR_E_UNKNOWN_NODE;
  const int b = e->batch_i;
  e->batch_i = (b + 1) % jr_engine::NBUF;
  jr_status st = batch_reserve(e, b, n);
  if (st != JR_OK) return st;
  CK(cudaMemcpyAsync(e->batch[b], proposals, n * sizeof(jr_proposal), cudaMemcpyHostToDevice, e->h2d));
  CK(cudaEventRecord(e->batch_ready[b], e->h2d));
  CK(cudaStreamWaitEvent(e->stream, e->batch_ready[b], 0));
  return batch_launch(e, b, now0, dt, n_steps);
}

jr_status jr_run_tokens(jr_engine* e, uint64_t now0, uint32_t dt, uint32_t n_steps, const uint64_t* tokens) {
  if (!e || !tokens) return JR_E_INVAL;
  if (n_steps == 0) return JR_OK;
  CK(cudaSetDevice(e->cfg.device));
  const uint32_t G = e->d.G;
  const size_t n = (size_t)n_steps * G;
  const int b = e->batch_i;
  e->batch_i = (b + 1) % jr_engine::NBUF;
  jr_status st = batch_reserve(e, b, n);  // batch_free[b] also covers tokbuf[b]: the routing kernel precedes the step
  if (st != JR_OK) return st;
  if (n > e->tok_cap[b]) {
    if (e->batch_used[b]) CK(cudaEventSynchronize(e->batch_free[b]));
    if (e->tokbuf[b]) cudaFree(e->tokbuf[b]);
    e->tokbuf[b] = nullptr;
    e->tok_cap[b] = 0;
    CK(cudaMalloc(&e->tokbuf[b], n * sizeof(unsigned long long)));
    e->tok_cap[b] = n;
  }
  CK(cudaMemcpyAsync(e->tokbuf[b], tokens, n * sizeof(unsigned long long), cudaMemcpyHostToDevice, e->h2d));
  CK(cudaEventRecord(e->batch_ready[b], e->h2d));
  CK(cudaStreamWaitEvent(e->stream, e->batch_ready[b], 0));
  // on the engine stream: ordered after the leader_table_kernel that last wrote `route`
  const unsigned blocks = (unsigned)std::min<size_t>((n + 255) / 256, (size_t)std::max(e->sms, 1u) * 16);
  JR_LAUNCH(route_tokens_kernel, blocks, 256, e->stream, e->tokbuf[b], e->route, e->batch[b], G, n);
  CK(cudaGetLastError());
  return batch_launch(e, b, now0, dt, n_steps);
}

jr_status jr_run_token_runs(jr_engine* e, uint64_t now0, uint32_t dt, uint32_t n_steps, const jr_token_run* runs) {
  if (!e || !runs) return JR_E_INVAL;
  if (n_steps == 0) return JR_OK;
  CK(cudaSetDevice(e->cfg.device));
  const uint32_t G = e->d.G;
  const int b = e->batch_i;
  e->batch_i = (b + 1) % jr_engine::NBUF;
  jr_status st = batch_reserve(e, b, G);   // batch[b] doubles as the staging buffer: G x 16 bytes
  if (st != JR_OK) return st;
  CK(cudaMemcpyAsync(e->batch[b], runs, (size_t)G * sizeof(jr_token_run), cudaMemcpyHostToDevice, e->h2d));
  CK(cudaEventRecord(e->batch_ready[b], e->h2d));
  CK(cudaStreamWaitEvent(e->stream, e->batch_ready[b], 0));
  StepParams p;
  p.now = now0;
  p.step_index = e->step_index;
  p.n_synth = 0;
  p.n_ticks = n_steps;
  p.dt = dt;
  p.cur = e->cur;
  p.proposals = nullptr;
  p.prop_stride = 0;
  p.tok_runs = reinterpret_cast<const uint4*>(e->batch[b]);
  p.tok_route = e->route;    // on the engine stream: ordered after the leader_table_kernel that last wrote it
  p.tok_tick = 0;
  p.phases = PH_RESET_OUT | PH_DRAIN | PH_PROPOSE | PH_TICK;
  p.trunc = e->auto_trunc ? 1u : 0u;
  p.trunc_margin = e->auto_trunc_margin;
  st = launch_step(e, p);
  if (st != JR_OK) return st;
  CK(cudaEventRecord(e->batch_free[b], e->stream));
  e->batch_used[b] = true;
  e->cur ^= (int)(n_steps & 1u);
  e->step_index += n_steps;
  return JR_OK;
}

jr_status jr_drain_fsm(jr_engine* e, jr_fsm_instr* out, size_t cap, size_t* n) {
  if (!e || !n) return JR_E_INVAL;
  CK(cudaSetDevice(e->cfg.device));
  if (!(e->d.flags & JR_F_CAPTURE_FSM)) { *n = 0; return JR_OK; }
  std::vector<jr_fsm_instr> fsm;
  jr_status st = capture_fsm(e, fsm);
  if (st != JR_OK && st != JR_E_CAPACITY) return st;
  *n = fsm.size();
  if (out) memcpy(out, fsm.data(), std::min(fsm.size(), cap) * sizeof(jr_fsm_instr));
  return ((out && fsm.size() > cap) || st == JR_E_CAPACITY) ? JR_E_CAPACITY : JR_OK;
}

jr_status jr_fsm_fold(const jr_fsm_record* recs, size_t n, uint32_t G, uint32_t R, uint32_t* applied_hi, uint64_t* totals) {
  if ((!recs && n) || !applied_hi || !totals || R < 1 || R > JR_MAX_REPLICAS) return JR_E_INVAL;
  uint64_t na = 0, nn = 0;
  for (size_t i = 0; i < n; ++i) {
    const jr_fsm_record& rc = recs[i];
    const uint32_t kind = JR_FSMR_KIND(rc.hdr), node = JR_FSMR_NODE(rc.hdr), count = JR_FSMR_COUNT(rc.hdr);
    if (rc.group >= G || node > R) return JR_E_INVAL;
    if (kind == JR_FSMR_APPLY) {
      if (rc.addr) {   // shared by the nodes of the mask
        if (rc.addr >> R) return JR_E_INVAL;
        for (uint32_t n = 0; n < R; ++n)
          if ((rc.addr >> n) & 1u) {
            uint32_t& hi = applied_hi[(size_t)n * G + rc.group];
            hi = std::max(hi, rc.id0 + count - 1);
            na += count;
          }
      } else {
        uint32_t& hi = applied_hi[(size_t)(node - 1) * G + rc.group];
        hi = std::max(hi, rc.id0 + count - 1);
        na += count;
      }
    } else if (kind == JR_FSMR_NOTIFY) {
      nn += count;
    }
  }
  totals[0] += na;
  totals[1] += nn;
  totals[2] += n;
  return JR_OK;
}

// jr_fsm_fold_mt: a small persistent pool (created on first use and deliberately never destroyed: its workers sleep on
// a condition variable for the life of the process).  A batch is sorted by (node, group); thread t folds the records of
// groups [G*t/T, G*(t+1)/T) of EVERY node section (found by binary search), so no two threads ever touch the same
// watermark -- masked records included, because all nodes of a group belong to the same thread -- and no atomics are
// needed.  A batch that is not sorted that way is folded on the calling thread.
namespace {
struct FoldJob {
  const jr_fsm_record* recs = nullptr;
  size_t n = 0;
  uint32_t G = 0, R = 0, parts = 0;
  uint32_t* applied = nullptr;
  size_t sec[JR_MAX_REPLICAS + 1];   // record index where node k+1's section starts
  uint64_t na[64], nn[64];
  int bad[64];
};
inline uint64_t rec_key(const jr_fsm_record& rc) { return ((uint64_t)JR_FSMR_NODE(rc.hdr) << 32) | rc.group; }
size_t lower_bound_key(const jr_fsm_record* recs, size_t lo, size_t hi, uint64_t key) {
  while (lo < hi) {
    const size_t mid = lo + (hi - lo) / 2;
    if (rec_key(recs[mid]) < key) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}
void fold_slice(FoldJob& j, uint32_t t) {
  const uint32_t g_lo = (uint32_t)((uint64_t)j.G * t / j.parts), g_hi = (uint32_t)((uint64_t)j.G * (t + 1) / j.parts);
  uint64_t na = 0, nn = 0;
  for (uint32_t node = 1; node <= j.R; ++node) {
    const size_t lo = lower_bound_key(j.recs, j.sec[node - 1], j.sec[node], ((uint64_t)node << 32) | g_lo);
    const size_t hi = lower_bound_key(j.recs, lo, j.sec[node], ((uint64_t)node << 32) | g_hi);
    for (size_t i = lo; i < hi; ++i) {
      const jr_fsm_record& rc = j.recs[i];
      const uint32_t kind = JR_FSMR_KIND(rc.hdr), count = JR_FSMR_COUNT(rc.hdr);
      if (kind == JR_FSMR_APPLY) {
        if (rc.addr) {
          if (rc.addr >> j.R) { j.bad[t] = 1; return; }
          for (uint32_t k = 0; k < j.R; ++k)
            if ((rc.addr >> k) & 1u) {
              uint32_t& hi_w = j.applied[(size_t)k * j.G + rc.group];
              hi_w = std::max(hi_w, rc.id0 + count - 1);
              na += count;
            }
        } else {
          uint32_t& hi_w = j.applied[(size_t)(node - 1) * j.G + rc.group];
          hi_w = std::max(hi_w, rc.id0 + count - 1);
          na += count;
        }
      } else if (kind == JR_FSMR_NOTIFY) {
        nn += count;
      }
    }
  }
  j.na[t] = na;
  j.nn[t] = nn;
}
class FoldPool {
  // Workers SPIN for a little while after a job before they go to sleep: a host that folds a batch every few hundred
  // microseconds (bench.py's end-to-end leg) then never pays the futex wake-up of seven threads -- which took as long as
  // the fold itself.  A host that folds rarely finds them asleep on the condition variable, as before.
  static constexpr long long SPIN_NS = 2'000'000;
 public:
  static FoldPool& get() { static FoldPool* p = new FoldPool(); return *p; }   // leaked on purpose (see above)
  void run(FoldJob& j) {
    {
      std::lock_guard<std::mutex> l(m_);
      while (n_workers_ + 1 < j.parts) {   // worker k serves slice k + 1; the caller folds slice 0
        const uint32_t k = n_workers_++;
        std::thread th([this, k] { loop(k); });
        th.detach();
      }
      job_ = &j;
      left_.store(j.parts - 1, std::memory_order_relaxed);
      // one word says which job is current and how many slices it has: a worker decides from a single load
      state_.store(((state_.load(std::memory_order_relaxed) >> 8) + 1) << 8 | j.parts, std::memory_order_release);
    }
    if (sleepers_.load(std::memory_order_acquire)) cv_.notify_all();
    fold_slice(j, 0);
    const auto t0 = std::chrono::steady_clock::now();
    while (left_.load(std::memory_order_acquire) != 0) {
      if (std::chrono::steady_clock::now() - t0 > std::chrono::nanoseconds(SPIN_NS)) {
        std::unique_lock<std::mutex> l(m_);
        done_.wait(l, [this] { return left_.load(std::memory_order_acquire) == 0; });
        break;
      }
      cpu_relax();
    }
  }
 private:
  static void cpu_relax() {
#if defined(__x86_64__) || defined(__i386__)
    __builtin_ia32_pause();
#endif
  }
  void loop(uint32_t k) {
    uint64_t seen = 0;   // generation (state >> 8) this worker has dealt with
    for (;;) {
      uint64_t st = state_.load(std::memory_order_acquire);
      const auto t0 = std::chrono::steady_clock::now();
      while ((st >> 8) == seen) {
        if (std::chrono::steady_clock::now() - t0 > std::chrono::nanoseconds(SPIN_NS)) {
          std::unique_lock<std::mutex> l(m_);
          sleepers_.fetch_add(1, std::memory_order_acq_rel);
          cv_.wait(l, [&] { return (state_.load(std::memory_order_acquire) >> 8) != seen; });
          sleepers_.fetch_sub(1, std::memory_order_acq_rel);
        } else {
          cpu_relax();
        }
        st = state_.load(std::memory_order_acquire);
      }
      seen = st >> 8;
      if (k + 1 >= (uint32_t)(st & 255u)) continue;   // not one of this job's slices (and then job_ is not this worker's to touch)
      fold_slice(*job_, k + 1);                         // (run() cannot return, nor the next job start, before left_ reaches 0)
      if (left_.fetch_sub(1, std::memory_order_acq_rel) == 1) {
        std::lock_guard<std::mutex> l(m_);
        done_.notify_all();
      }
    }
  }
  std::mutex m_;
  std::condition_variable cv_, done_;
  uint32_t n_workers_ = 0;
  FoldJob* job_ = nullptr;
  std::atomic<uint32_t> left_{0}, sleepers_{0};
  std::atomic<uint64_t> state_{0};   // generation << 8 | slices of the current job
};
}  // namespace

jr_status jr_fsm_fold_mt(const jr_fsm_record* recs, size_t n, uint32_t G, uint32_t R, uint32_t* applied_hi, uint64_t* totals,
                         uint32_t n_threads) {
  if (n_threads <= 1 || n < 4096) return jr_fsm_fold(recs, n, G, R, applied_hi, totals);
  if ((!recs && n) || !applied_hi || !totals || R < 1 || R > JR_MAX_REPLICAS) return JR_E_INVAL;
  FoldJob j;
  j.recs = recs; j.n = n; j.G = G; j.R = R; j.applied = applied_hi;
  j.parts = std::min<uint32_t>(n_threads, 64);
  // node sections; then a cheap sortedness probe (a full check would cost as much as the fold)
  j.sec[0] = 0;
  for (uint32_t node = 1; node <= R; ++node) j.sec[node] = lower_bound_key(recs, j.sec[node - 1], n, (uint64_t)(node + 1) << 32);
  bool sorted = j.sec[R] == n && recs[n - 1].group < G;
  for (size_t probe = 1; sorted && probe < 64; ++probe) {
    const size_t i = n * probe / 64;
    sorted = i == 0 || rec_key(recs[i - 1]) <= rec_key(recs[i]);
  }
  if (!sorted) return jr_fsm_fold(recs, n, G, R, applied_hi, totals);
  static std::mutex* one_at_a_time = new std::mutex();
  std::lock_guard<std::mutex> guard(*one_at_a_time);
  for (uint32_t t = 0; t < j.parts; ++t) { j.na[t] = j.nn[t] = 0; j.bad[t] = 0; }
  FoldPool::get().run(j);
  for (uint32_t t = 0; t < j.parts; ++t) {
    if (j.bad[t]) return JR_E_INVAL;
    totals[0] += j.na[t];
    totals[1] += j.nn[t];
  }
  totals[2] += n;
  return JR_OK;
}

jr_status jr_fsm_records_async(jr_engine* e) {
  if (!e) return JR_E_INVAL;
  CK(cudaSetDevice(e->cfg.device));
  return fsm_records_enqueue(e);
}

jr_status jr_fsm_records_wait(jr_engine* e, const jr_fsm_record** records, jr_fsm_batch* batch) {
  if (!e) return JR_E_INVAL;
  CK(cudaSetDevice(e->cfg.device));   // (may be a consumer thread of its own: the device is per thread)
  return fsm_records_take(e, records, batch);
}

jr_status jr_fsm_responses(jr_engine* e, const jr_fsm_record** responses, jr_fsm_batch* batch) {
  if (!e) return JR_E_INVAL;
  if (!e->resp_cap) { set_err("engine created without JR_F_CLIENT_RESPONSES"); return JR_E_INVAL; }
  int b;
  { std::lock_guard<std::mutex> l(e->qmu); b = e->resp_b; }
  if (b < 0) { set_err("no batch has been taken yet"); return JR_E_INVAL; }
  const FsmHeader& h = e->fsm_host_hdr[b][1];
  if (responses) *responses = reinterpret_cast<const jr_fsm_record*>(e->fsm_host[b] + 2 * (size_t)e->fsm_cap);
  if (batch) {
    memset(batch, 0, sizeof *batch);
    batch->n_records = h.n_records;
    batch->n_dropped = h.n_dropped;
    batch->n_instructions = h.n_instructions;
    for (uint32_t r = 0; r <= JR_MAX_REPLICAS; ++r) batch->node_offset[r] = r <= e->d.R ? h.node_offset[r] : h.node_offset[e->d.R];
  }
  if (h.n_dropped) {
    set_err("%llu notifications / responses were dropped (JR_NOTIFY_RUNS, fsm_units or lost records)", (unsigned long long)h.n_dropped);
    return JR_E_CAPACITY;
  }
  return JR_OK;
}

// Pure host code: records -> Instructions (include/josefine_raft_abi.h, jr_fsm_record).
jr_status jr_fsm_expand(const jr_fsm_record* recs, size_t n_records, uint32_t G, uint32_t R, jr_fsm_instr* out, size_t cap,
                        size_t* n_out) {
  if (!n_out || (!recs && n_records) || R < 1 || R > JR_MAX_REPLICAS || G < 1) return JR_E_INVAL;
  // stable counting sort of record indices by (group, node).  An APPLY record with a node mask (addr != 0: symmetric
  // followers share it) goes into the bucket of every node of the mask, in front of that node's own records: masked
  // records are only ever produced while the nodes' own streams are still empty.
  const size_t nb = (size_t)G * R;
  std::vector<uint32_t> start(nb + 1, 0u);
  auto masked = [&](const jr_fsm_record& rc) { return JR_FSMR_KIND(rc.hdr) == JR_FSMR_APPLY && rc.addr != 0; };
  for (size_t i = 0; i < n_records; ++i) {
    const uint32_t node = JR_FSMR_NODE(recs[i].hdr);
    if (recs[i].group >= G || node > R || JR_FSMR_KIND(recs[i].hdr) > JR_FSMR_PATTERN) return JR_E_INVAL;
    if (masked(recs[i])) {
      if (recs[i].addr >> R) return JR_E_INVAL;
      for (uint32_t n = 0; n < R; ++n)
        if ((recs[i].addr >> n) & 1u) ++start[(size_t)recs[i].group * R + n + 1];
    } else {
      ++start[(size_t)recs[i].group * R + (node - 1) + 1];
    }
  }
  for (size_t b = 0; b < nb; ++b) start[b + 1] += start[b];
  std::vector<uint32_t> order(start[nb]), fill(start.begin(), start.end() - 1);
  for (int pass = 0; pass < 2; ++pass)
    for (size_t i = 0; i < n_records; ++i) {
      if (masked(recs[i]) != (pass == 0)) continue;
      if (pass == 0) {
        for (uint32_t n = 0; n < R; ++n)
          if ((recs[i].addr >> n) & 1u) order[fill[(size_t)recs[i].group * R + n]++] = (uint32_t)i;
      } else {
        order[fill[(size_t)recs[i].group * R + (JR_FSMR_NODE(recs[i].hdr) - 1)]++] = (uint32_t)i;
      }
    }
  size_t k = 0;
  std::vector<uint64_t> is_notify;
  for (size_t b = 0; b < nb; ++b) {
    const uint32_t lo = start[b], hi = start[b + 1];
    if (lo == hi) continue;
    const uint32_t g = (uint32_t)(b / R), node = (uint32_t)(b % R) + 1;
    size_t n_apply = 0, n_note = 0;
    for (uint32_t j = lo; j < hi; ++j) {
      const jr_fsm_record& rc = recs[order[j]];
      if (JR_FSMR_KIND(rc.hdr) == JR_FSMR_APPLY) n_apply += JR_FSMR_COUNT(rc.hdr);
      else if (JR_FSMR_KIND(rc.hdr) == JR_FSMR_NOTIFY) n_note += JR_FSMR_COUNT(rc.hdr);
    }
    const size_t total = n_apply + n_note;
    is_notify.assign((total + 63) / 64, 0ull);
    size_t marked = 0;
    for (uint32_t j = lo; j < hi; ++j) {
      const jr_fsm_record& rc = recs[order[j]];
      if (JR_FSMR_KIND(rc.hdr) != JR_FSMR_PATTERN) continue;
      const uint32_t nbits = JR_FSMR_COUNT(rc.hdr);
      if (nbits > 160) return JR_E_INVAL;
      for (uint32_t bit = 0; bit < nbits; ++bit)
        if ((bit < 64 ? rc.tok0 >> bit : bit < 128 ? rc.stride >> (bit - 64) : (uint64_t)rc.addr >> (bit - 128)) & 1ull) {
          const size_t pos = (size_t)rc.id0 + bit;
          if (pos >= total || ((is_notify[pos >> 6] >> (pos & 63)) & 1ull)) return JR_E_INVAL;
          is_notify[pos >> 6] |= 1ull << (pos & 63);
          ++marked;
        }
    }
    if (marked != n_note) return JR_E_INVAL;
    // two cursors, one per kind, both in record order
    uint32_t ja = lo, jn = lo, ia = 0, in_ = 0;
    for (size_t pos = 0; pos < total; ++pos) {
      const bool note = (is_notify[pos >> 6] >> (pos & 63)) & 1ull;
      uint32_t& j = note ? jn : ja;
      uint32_t& i = note ? in_ : ia;
      const uint32_t want = note ? JR_FSMR_NOTIFY : JR_FSMR_APPLY;
      while (JR_FSMR_KIND(recs[order[j]].hdr) != want || i >= JR_FSMR_COUNT(recs[order[j]].hdr)) { ++j; i = 0; }
      const jr_fsm_record& rc = recs[order[j]];
      if (out && k < cap) {
        jr_fsm_instr f;
        memset(&f, 0, sizeof f);
        f.group = g;
        f.node = node;
        if (note) {
          f.kind = JR_FSM_NOTIFY;
          f.client_kind = (uint8_t)(rc.addr >> 16);
          f.client_id = rc.addr & 0xffffu;
          f.block = jr_block{(uint64_t)(rc.id0 + i), 0, rc.tok0 + (uint64_t)i * rc.stride};
        } else {
          f.kind = JR_FSM_APPLY;
          const uint32_t bid = rc.id0 + i;
          if (JR_FSMR_COUNT(rc.hdr) == 1) f.block = jr_block{bid, (uint32_t)rc.stride, rc.tok0};
          else f.block = jr_block{bid, bid - 1u, rc.tok0 + (uint64_t)i * rc.stride};
        }
        out[k] = f;
      }
      ++k;
      ++i;
    }
  }
  *n_out = k;
  return (out && k > cap) || (!out && k) ? JR_E_CAPACITY : JR_OK;
}

// ---- introspection ----------------------------------------------------------------------------

// Device scratch that grows on demand (contents are not kept).
static jr_status scratch_reserve(void** buf, size_t* cap, size_t bytes) {
  if (bytes <= *cap) return JR_OK;
  if (*buf) cudaFree(*buf);
  *buf = nullptr;
  *cap = 0;
  const size_t want = std::max<size_t>(bytes * 2, 4096);
  CK(cudaMalloc(buf, want));
  *cap = want;
  return JR_OK;
}

static jr_status many_reserve(jr_engine* e, size_t bytes) { return scratch_reserve(&e->many_buf, &e->many_cap, bytes); }

jr_status jr_query_many(jr_engine* e, const uint32_t* groups, const uint32_t* nodes, size_t n, jr_replica_state* out) {
  if (!e || !out || !groups || !nodes) return JR_E_INVAL;
  if (n == 0) return JR_OK;
  if (n > 0x7fffffffu) return JR_E_INVAL;
  for (size_t i = 0; i < n; ++i)
    if (groups[i] >= e->d.G || nodes[i] < 1 || nodes[i] > e->d.R) return JR_E_INVAL;
  CK(cudaSetDevice(e->cfg.device));
  const size_t idx = ((n * 2 * sizeof(uint32_t)) + 15) / 16 * 16;   // [groups][nodes] then the states
  jr_status st = many_reserve(e, idx + n * sizeof(jr_replica_state));
  if (st != JR_OK) return st;
  uint32_t* dg = (uint32_t*)e->many_buf;
  uint32_t* dn = dg + n;
  jr_replica_state* ds = (jr_replica_state*)((char*)e->many_buf + idx);
  CK(cudaMemcpyAsync(dg, groups, n * sizeof(uint32_t), cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemcpyAsync(dn, nodes, n * sizeof(uint32_t), cudaMemcpyHostToDevice, e->stream));
  JR_LAUNCH(query_kernel, (unsigned)((n + 127) / 128), 128, e->stream, e->d, dg, dn, (uint32_t)n, ds);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out, ds, n * sizeof(jr_replica_state), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return JR_OK;
}

jr_status jr_query(jr_engine* e, uint32_t group, uint32_t node, jr_replica_state* out) {
  return jr_query_many(e, &group, &node, 1, out);
}

jr_status jr_chain_read_many(jr_engine* e, const uint32_t* groups, const uint32_t* nodes, const uint64_t* first_id,
                             const uint32_t* count, size_t n, jr_block* out, uint8_t* present) {
  if (!e || !groups || !nodes || !first_id || !count) return JR_E_INVAL;
  if (n == 0) return JR_OK;
  if (n > 0x7fffffffu) return JR_E_INVAL;
  std::vector<uint4> reqs(n);
  size_t total = 0;
  for (size_t i = 0; i < n; ++i) {
    if (groups[i] >= e->d.G || nodes[i] < 1 || nodes[i] > e->d.R) return JR_E_INVAL;
    if (first_id[i] > 0xffffffffull - count[i]) return JR_E_INVAL;   // ids past 2^32-2 (no wrap: count < 2^32)
    reqs[i] = make_uint4(groups[i], nodes[i] - 1, (uint32_t)first_id[i], (uint32_t)total);
    total += count[i];
    if (total > 0xffffffffull) return JR_E_INVAL;
  }
  if (total == 0) return JR_OK;
  CK(cudaSetDevice(e->cfg.device));
  const size_t o_cnt = n * sizeof(uint4), o_blk = (o_cnt + n * sizeof(uint32_t) + 15) / 16 * 16;
  const size_t o_pre = o_blk + total * sizeof(jr_block);
  jr_status st = many_reserve(e, o_pre + total);
  if (st != JR_OK) return st;
  char* base = (char*)e->many_buf;
  CK(cudaMemcpyAsync(base, reqs.data(), n * sizeof(uint4), cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemcpyAsync(base + o_cnt, count, n * sizeof(uint32_t), cudaMemcpyHostToDevice, e->stream));
  JR_LAUNCH(chain_read_kernel, (unsigned)n, 128, e->stream, e->d, (const uint4*)base, (const uint32_t*)(base + o_cnt),
            (jr_block*)(base + o_blk), (uint8_t*)(base + o_pre));
  CK(cudaGetLastError());
  if (out) CK(cudaMemcpyAsync(out, base + o_blk, total * sizeof(jr_block), cudaMemcpyDeviceToHost, e->stream));
  if (present) CK(cudaMemcpyAsync(present, base + o_pre, total, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));   // also covers `reqs`, which lives on this stack
  return JR_OK;
}

jr_status jr_chain_read(jr_engine* e, uint32_t group, uint32_t node, uint64_t first, uint32_t n, jr_block* out,
                        uint8_t* present) {
  if (n == 0) return (!e || group >= e->d.G || node < 1 || node > e->d.R) ? JR_E_INVAL : JR_OK;
  return jr_chain_read_many(e, &group, &node, &first, &n, 1, out, present);
}

jr_status jr_state_digest(jr_engine* e, uint64_t* out) {
  if (!e || !out) return JR_E_INVAL;
  CK(cudaSetDevice(e->cfg.device));
  const size_t plane = (size_t)e->d.R * e->d.Gp;
  CK(cudaMemsetAsync(e->scratch, 0, 8 * sizeof(unsigned long long), e->stream));
  JR_LAUNCH(state_digest_kernel, (unsigned)((plane + CTA_THREADS - 1) / CTA_THREADS), CTA_THREADS, e->stream, e->d, e->scratch);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out, e->scratch, sizeof(uint64_t), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return JR_OK;
}

static jr_status stream_sums(jr_engine* e, uint64_t v[5]) {
  CK(cudaSetDevice(e->cfg.device));
  const size_t plane = (size_t)e->d.R * e->d.Gp;
  CK(cudaMemsetAsync(e->scratch, 0, 8 * sizeof(unsigned long long), e->stream));
  JR_LAUNCH(stream_digest_kernel, (unsigned)((plane + CTA_THREADS - 1) / CTA_THREADS), CTA_THREADS, e->stream, e->d, e->scratch);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(v, e->scratch, 5 * sizeof(uint64_t), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return JR_OK;
}

jr_status jr_stream_digest(jr_engine* e, uint64_t* md, uint64_t* fd, uint64_t* nm, uint64_t* nf) {
  if (!e) return JR_E_INVAL;
  if (!(e->d.flags & JR_F_STREAM_DIGEST)) { set_err("engine created without JR_F_STREAM_DIGEST"); return JR_E_INVAL; }
  uint64_t v[5];
  jr_status st = stream_sums(e, v);
  if (st != JR_OK) return st;
  if (md) *md = v[0];
  if (fd) *fd = v[1];
  if (nm) *nm = v[2];
  if (nf) *nf = v[3];
  return JR_OK;
}

jr_status jr_fold_count(jr_engine* e, uint64_t* n) {
  if (!e || !n) return JR_E_INVAL;
  *n = 0;
  if (!e->last_launch_folded) return JR_OK;
  CK(cudaSetDevice(e->cfg.device));
  std::vector<uint8_t> h(e->d.Gp);
  CK(cudaMemcpyAsync(h.data(), e->symdone, h.size(), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  for (uint32_t g = 0; g < e->d.G; ++g) *n += h[g];
  return JR_OK;
}

jr_status jr_fault_count(jr_engine* e, uint64_t* n) {
  if (!e || !n) return JR_E_INVAL;
  uint64_t v[5];
  jr_status st = stream_sums(e, v);
  if (st != JR_OK) return st;
  *n = v[4];
  return JR_OK;
}

// ---- maintenance ------------------------------------------------------------------------------

jr_status jr_compact(jr_engine* e) {
  if (!e) return JR_E_INVAL;
  CK(cudaSetDevice(e->cfg.device));
  const size_t plane = (size_t)e->d.R * e->d.Gp;
  JR_LAUNCH(compact_kernel, (unsigned)((plane + 127) / 128), 128, e->stream, e->d);
  CK(cudaGetLastError());
  return JR_OK;
}

jr_status jr_truncate(jr_engine* e, uint32_t margin) {
  if (!e) return JR_E_INVAL;
  CK(cudaSetDevice(e->cfg.device));
  JR_LAUNCH(truncate_kernel, (e->d.Gp + 127) / 128, 128, e->stream, e->d, margin, (const uint8_t*)nullptr);
  CK(cudaGetLastError());
  return JR_OK;
}

jr_status jr_host_alloc(size_t bytes, void** out) {
  if (!out || !bytes) return JR_E_INVAL;
  *out = nullptr;
  cudaError_t err = cudaHostAlloc(out, bytes, 0);
  if (err != cudaSuccess) {
    set_err("cudaHostAlloc(%zu bytes): %s", bytes, cudaGetErrorString(err));
    return err == cudaErrorMemoryAllocation ? JR_E_NOMEM : JR_E_CUDA;
  }
  return JR_OK;
}

void jr_host_free(void* p) {
  if (p) cudaFreeHost(p);
}

jr_status jr_set_auto_truncate(jr_engine* e, int enabled, uint32_t margin) {
  if (!e) return JR_E_INVAL;
  e->auto_trunc = enabled != 0;
  e->auto_trunc_margin = margin;
  return JR_OK;
}

jr_status jr_chain_export_many(jr_engine* e, const uint32_t* groups, const uint32_t* nodes, size_t n,
                               jr_persisted_chain* out, jr_block* blocks, size_t cap_blocks, size_t* n_blocks) {
  if (!e || !n_blocks || (n && (!groups || !nodes || !out))) return JR_E_INVAL;
  *n_blocks = 0;
  if (n == 0) return JR_OK;
  if (n > 0x7fffffffu) return JR_E_INVAL;
  std::vector<uint2> targets(n);
  for (size_t k = 0; k < n; ++k) {
    if (groups[k] >= e->d.G || nodes[k] < 1 || nodes[k] > e->d.R) {
      set_err("target %zu: group or node out of range", k);
      return JR_E_INVAL;
    }
    targets[k] = make_uint2(groups[k], nodes[k] - 1);
  }
  CK(cudaSetDevice(e->cfg.device));
  // pass 1: descriptors with counts -> host.  The scan over the counts runs here: the descriptors have to reach the
  // caller anyway, and the call synchronises, so a device scan would save no round trip.
  const size_t o_desc = (n * sizeof(uint2) + 15) / 16 * 16;
  jr_status st = many_reserve(e, o_desc + n * sizeof(jr_persisted_chain));
  if (st != JR_OK) return st;
  char* base = (char*)e->many_buf;
  CK(cudaMemcpyAsync(base, targets.data(), n * sizeof(uint2), cudaMemcpyHostToDevice, e->stream));
  JR_LAUNCH(export_count_kernel, (unsigned)((n + 127) / 128), 128, e->stream, e->d, (const uint2*)base, (uint32_t)n,
            (jr_persisted_chain*)(base + o_desc));
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out, base + o_desc, n * sizeof(jr_persisted_chain), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));   // (also covers `targets`, which lives on this stack)
  uint64_t total = 0;
  for (size_t k = 0; k < n; ++k) {
    out[k].first_block = total;
    total += out[k].n_blocks;
  }
  *n_blocks = (size_t)total;
  if (!blocks || cap_blocks < total) return JR_E_CAPACITY;
  if (total == 0) return JR_OK;
  // pass 2: the blocks, packed in request order into a staging buffer, then one copy out
  const size_t o_blk = (n * sizeof(jr_persisted_chain) + 15) / 16 * 16;
  if ((st = many_reserve(e, o_blk + total * sizeof(jr_block))) != JR_OK) return st;
  base = (char*)e->many_buf;
  CK(cudaMemcpyAsync(base, out, n * sizeof(jr_persisted_chain), cudaMemcpyHostToDevice, e->stream));
  JR_LAUNCH(export_pack_kernel, (unsigned)((n + 127) / 128), 128, e->stream, e->d, (const jr_persisted_chain*)base,
            (uint32_t)n, (jr_block*)(base + o_blk));
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(blocks, base + o_blk, total * sizeof(jr_block), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return JR_OK;
}

jr_status jr_node_restart_many(jr_engine* e, uint64_t now_ms, const jr_persisted_chain* chains, size_t n,
                               const jr_block* blocks, size_t n_blocks) {
  if (!e || (n && !chains) || (n_blocks && !blocks)) return JR_E_INVAL;
  if (n == 0) return JR_OK;
  if (n > 0x7fffffffu) return JR_E_INVAL;
  const Dev& d = e->d;
  // everything is checked before the first device write: on JR_E_INVAL the engine is untouched
  uint32_t g_lo = 0xffffffffu, g_hi = 0;   // the groups the call names lie in [g_lo, g_hi]
  for (size_t k = 0; k < n; ++k) {
    if (chains[k].group >= d.G || chains[k].node < 1 || chains[k].node > d.R) {
      set_err("chains[%zu]: group or node out of range", k);
      return JR_E_INVAL;
    }
    g_lo = std::min(g_lo, chains[k].group);
    g_hi = std::max(g_hi, chains[k].group);
  }
  const size_t span = (size_t)g_hi - g_lo + 1;
  std::vector<uint8_t> seen(span * d.R, 0);
  bool host_blocks = false;
  for (size_t k = 0; k < n; ++k) {
    const jr_persisted_chain& c = chains[k];
    uint8_t& s = seen[(size_t)(c.node - 1) * span + (c.group - g_lo)];
    if (s) {
      set_err("chains[%zu]: replica (%u, %u) appears twice", k, c.group, c.node);
      return JR_E_INVAL;
    }
    s = 1;
    if (c.n_blocks == JR_RESTART_IN_PLACE) continue;
    if (c.n_blocks > d.cap || c.first_block > n_blocks || n_blocks - c.first_block < c.n_blocks || c.commit >= JR_BLOCK_ID_LIMIT) {
      set_err("chains[%zu]: slice outside blocks[0, %zu), more than chain_capacity blocks, or commit >= 2^31 (D4)", k, n_blocks);
      return JR_E_INVAL;
    }
    host_blocks |= c.n_blocks > 0;
  }
  CK(cudaSetDevice(e->cfg.device));
  if (host_blocks) {
    std::vector<uint32_t> floor(span);   // the groups' floors: one copy of the TB plane's [g_lo, g_hi]
    CK(cudaMemcpyAsync(floor.data(), d.tb + g_lo, span * sizeof(uint32_t), cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
    for (size_t k = 0; k < n; ++k) {
      const jr_persisted_chain& c = chains[k];
      if (c.n_blocks == JR_RESTART_IN_PLACE) continue;
      const uint64_t lo = floor[c.group - g_lo];
      for (uint32_t j = 0; j < c.n_blocks; ++j) {
        const jr_block& b = blocks[c.first_block + j];
        if (b.id < lo || b.id - lo >= d.cap || b.id >= JR_BLOCK_ID_LIMIT || b.next >= JR_BLOCK_ID_LIMIT ||
            (j && b.id <= blocks[c.first_block + j - 1].id)) {
          set_err("chains[%zu] block %u: id not ascending, outside [floor, floor + chain_capacity) or >= 2^31, or next >= 2^31 (D4, D7)", k, j);
          return JR_E_INVAL;
        }
      }
    }
  }
  const size_t o_blk = (n * sizeof(jr_persisted_chain) + 15) / 16 * 16;
  jr_status st = many_reserve(e, o_blk + n_blocks * sizeof(jr_block));
  if (st != JR_OK) return st;
  char* base = (char*)e->many_buf;
  CK(cudaMemcpyAsync(base, chains, n * sizeof(jr_persisted_chain), cudaMemcpyHostToDevice, e->stream));
  if (n_blocks) CK(cudaMemcpyAsync(base + o_blk, blocks, n_blocks * sizeof(jr_block), cudaMemcpyHostToDevice, e->stream));
  JR_LAUNCH(node_restart_kernel, (unsigned)((n + 127) / 128), 128, e->stream, d, now_ms, (const jr_persisted_chain*)base,
            (uint32_t)n, (const jr_block*)(base + o_blk), e->rp.rm);
  CK(cudaGetLastError());
  if (d.lqm) {
    JR_LAUNCH(link_queues_mask_kernel, (unsigned)((n + 127) / 128), 128, e->stream, d, (const jr_persisted_chain*)base, (uint32_t)n);
    CK(cudaGetLastError());
  }
  CK(cudaStreamSynchronize(e->stream));
  return JR_OK;
}

// One replica: a one-element jr_node_restart_many.  `blocks` may come in any order and repeat an id; the table holds
// the last copy of each id, so they are sorted stably and all but the last copy dropped first.
jr_status jr_node_restart(jr_engine* e, uint32_t group, uint32_t node, uint64_t now_ms, const jr_block* blocks,
                          size_t n_blocks, uint64_t commit, int commit_key) {
  if (!e || group >= e->d.G || node < 1 || node > e->d.R || (n_blocks && !blocks)) return JR_E_INVAL;
  if (n_blocks > e->d.cap || commit >= JR_BLOCK_ID_LIMIT) return JR_E_INVAL;
  std::vector<jr_block> v(blocks, blocks + n_blocks);
  std::stable_sort(v.begin(), v.end(), [](const jr_block& a, const jr_block& b) { return a.id < b.id; });
  size_t m = 0;
  for (size_t k = 0; k < v.size(); ++k)
    if (k + 1 == v.size() || v[k + 1].id != v[k].id) v[m++] = v[k];
  jr_persisted_chain c;
  c.group = group;
  c.node = node;
  c.commit = commit;
  c.first_block = 0;
  c.n_blocks = (uint32_t)m;
  c.commit_key = commit_key ? 1u : 0u;
  return jr_node_restart_many(e, now_ms, &c, 1, v.data(), m);
}

jr_status jr_verify_groups(jr_engine* e, const uint32_t* groups, size_t n_groups, jr_verify_report* report,
                           jr_verify_finding* findings, size_t cap, size_t* n_findings) {
  if (!e || !report || !n_findings || (n_groups && !groups)) return JR_E_INVAL;
  const Dev& d = e->d;
  const size_t n = groups ? n_groups : d.G;
  std::vector<uint32_t> list;
  if (groups) {   // checked before the first device call: on JR_E_INVAL the engine is untouched
    std::vector<uint8_t> seen(d.G, 0);
    for (size_t k = 0; k < n; ++k) {
      if (groups[k] >= d.G || seen[groups[k]]) {
        set_err("groups[%zu]: out of range or named twice", k);
        return JR_E_INVAL;
      }
      seen[groups[k]] = 1;
    }
    list.assign(groups, groups + n);
    std::sort(list.begin(), list.end());   // findings come out in list order
  }
  memset(report, 0, sizeof *report);
  report->groups_checked = n;
  *n_findings = 0;
  if (n == 0) return JR_OK;
  CK(cudaSetDevice(e->cfg.device));
  const uint32_t T = CTA_THREADS;
  const size_t reps = (size_t)d.R * n;
  const uint32_t n_ctas = (uint32_t)((n + T - 1) / T);
  const size_t o_part = 16 * sizeof(unsigned long long), o_list = o_part + ((size_t)n_ctas * 8 + 15) / 16 * 16;
  const size_t o_vw = o_list + (n * 4 + 15) / 16 * 16, o_vf = o_vw + reps * sizeof(uint2);
  jr_status st = scratch_reserve(&e->verify_buf, &e->verify_cap, o_vf + reps * sizeof(uint2));
  if (st != JR_OK) return st;
  char* base = (char*)e->verify_buf;
  unsigned long long* rep = (unsigned long long*)base;
  unsigned long long* part = (unsigned long long*)(base + o_part);
  const uint32_t* dlist = groups ? (const uint32_t*)(base + o_list) : nullptr;   // null: group = list index
  uint2* vw = (uint2*)(base + o_vw);
  uint2* vf = (uint2*)(base + o_vf);
  CK(cudaMemsetAsync(rep, 0, VERIFY_COUNTS * sizeof(unsigned long long), e->stream));
  if (groups) CK(cudaMemcpyAsync(base + o_list, list.data(), n * 4, cudaMemcpyHostToDevice, e->stream));
  const unsigned grid = (unsigned)((reps + T - 1) / T);
  JR_LAUNCH(verify_walk_kernel, grid, T, e->stream, d, dlist, (uint32_t)n, vw);
  CK(cudaGetLastError());
  JR_LAUNCH(verify_judge_kernel, grid, T, e->stream, d, dlist, (uint32_t)n, (const uint2*)vw, vf, rep);
  CK(cudaGetLastError());
  unsigned long long cnt[VERIFY_COUNTS];
  CK(cudaMemcpyAsync(cnt, rep, sizeof cnt, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));   // (also covers `list`)
  report->replicas_checked = cnt[0];
  report->replicas_skipped = cnt[1];
  report->below_floor = cnt[2];
  report->commit_absent = cnt[3];
  report->chain_broken = cnt[4];
  report->diverged = cnt[5];
  report->leader_conflicts = cnt[6];
  const size_t total = (size_t)(cnt[2] + cnt[3] + cnt[4] + cnt[5] + cnt[6]);
  *n_findings = total;
  if (total == 0) return JR_OK;
  if (!findings || cap < total) return JR_E_CAPACITY;
  // something to report: count, scan and pack the findings in (group, node) order on the device, then one copy
  if ((st = many_reserve(e, total * sizeof(jr_verify_finding))) != JR_OK) return st;
  jr_verify_finding* out = (jr_verify_finding*)e->many_buf;
  JR_LAUNCH(verify_count_kernel, n_ctas, T, e->stream, d, (uint32_t)n, (const uint2*)vf, part);
  CK(cudaGetLastError());
  JR_LAUNCH(verify_scan_kernel, 1, 1, e->stream, part, n_ctas);
  CK(cudaGetLastError());
  JR_LAUNCH(verify_pack_kernel, n_ctas, T, e->stream, d, dlist, (uint32_t)n, (const uint2*)vf, (const unsigned long long*)part, out);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(findings, out, total * sizeof(jr_verify_finding), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return JR_OK;
}

// ---- checkpoint -----------------------------------------------------------------------------------
namespace {
struct SaveHeader {
  uint64_t magic, bytes;
  jr_config cfg;
  uint32_t cur, route_valid;
  uint64_t step_index;
};
constexpr uint64_t SAVE_MAGIC = 0x4a52454e47494e32ull;  // "JRENGIN2"
// Every allocation that holds the state of a group, in checkpoint order, and how a group image carries its share of it.
// jr_engine_save writes each one whole; jr_group_export carries each listed group's part of each one.  (The allocations
// that are neither -- transient scratch and engine-wide state -- are listed in DESIGN.md section 3f.)
enum class Carry : uint8_t {
  WORDS,        // word for word in the fixed record: per replica, or per group (per_group)
  TABLE,        // cnext / ctok: the rows present in the window
  MAIL,         // ob[0..1] / oc[0..1]: the previous step's mailbox, moved to the destination's parity
  FIFO,         // fs: the records fc counts
  NOTIFY_RUNS,  // the PN runs pnc counts
};
struct PlaneDesc {
  void* p;
  size_t bytes;                    // the checkpoint segment
  Carry carry;
  uint32_t words = 0, depth = 1;   // WORDS: 32-bit words per entry, entries per replica / group
  bool per_group = false;
};
std::vector<PlaneDesc> engine_planes(jr_engine* e) {
  const Dev& d = e->d;
  const size_t plane = (size_t)d.R * d.Gp;
  const size_t rows = (size_t)d.capm + 1;
  const uint32_t pq = (d.R + 3) / 4;
  std::vector<PlaneDesc> v = {
      {d.p0, plane * sizeof(uint4), Carry::WORDS, 4}, {d.p1, plane * sizeof(uint4), Carry::WORDS, 4},
      {d.p2, plane * sizeof(uint4), Carry::WORDS, 4}, {d.p3, plane * sizeof(uint4), Carry::WORDS, 4},
      {d.pr, plane * pq * sizeof(uint4), Carry::WORDS, 4, pq}, {d.mk, plane * sizeof(uint32_t), Carry::WORDS, 1},
      {d.qt, plane * JR_CLIENT_QUEUE_CAP * sizeof(uint4), Carry::WORDS, 4, JR_CLIENT_QUEUE_CAP},
      {d.dg, plane * sizeof(uint4), Carry::WORDS, 4}, {d.cn, plane * sizeof(uint2), Carry::WORDS, 2},
      {d.cnext, plane * rows * sizeof(uint32_t), Carry::TABLE}, {d.ctok, plane * rows * sizeof(unsigned long long), Carry::TABLE},
      {d.ob[0], plane * (size_t)d.U * sizeof(uint4), Carry::MAIL}, {d.ob[1], plane * (size_t)d.U * sizeof(uint4), Carry::MAIL},
      {d.oc[0], plane * sizeof(uint32_t), Carry::MAIL}, {d.oc[1], plane * sizeof(uint32_t), Carry::MAIL},
      {d.fs, plane * ((d.flags & JR_F_CAPTURE_FSM) ? 2 * (size_t)d.F : 1) * sizeof(uint4), Carry::FIFO},
      {d.fc, plane * sizeof(uint2), Carry::WORDS, 2},
      {d.tb, (size_t)d.Gp * sizeof(uint32_t), Carry::WORDS, 1, 1, true},
      {e->route, (size_t)d.G * sizeof(uint32_t), Carry::WORDS, 1, 1, true}};
  if (e->rp.pn) {   // the fsm::Driver maps (JR_F_CLIENT_RESPONSES only: other checkpoints keep their size and bytes)
    // one allocation, three consecutive segments: runs, run counts (u32, padded to 16 bytes), restart marks
    v.push_back({e->rp.pn, 2 * (size_t)JR_NOTIFY_RUNS * plane * sizeof(uint4), Carry::NOTIFY_RUNS});
    v.push_back({e->rp.pnc, (plane + 3) / 4 * sizeof(uint4), Carry::WORDS, 1});
    v.push_back({e->rp.rm, plane * sizeof(uint4), Carry::WORDS, 4});
  }
  if (d.links)   // the link matrices (JR_F_PEER_LINKS only, for the same reason)
    v.push_back({d.links, (size_t)d.Gp * sizeof(unsigned long long), Carry::WORDS, 2, 1, true});
  if (d.lq) {    // the link queues (JR_F_LINK_QUEUES only): non-empty masks, counts, units
    const uint32_t slots = std::max<uint32_t>(d.R - 1, 1u);
    v.push_back({d.lqm, (size_t)d.Gp * sizeof(unsigned long long), Carry::WORDS, 2, 1, true});
    v.push_back({d.lqc, plane * slots * sizeof(uint32_t), Carry::WORDS, 1, slots});
    v.push_back({d.lq, plane * slots * LQ_UNITS * sizeof(uint4), Carry::WORDS, 4, slots * LQ_UNITS});
  }
  return v;
}

// One group's link queues, as a checkpoint or an image holds them: every depth <= JR_LINK_QUEUE_MSGS, every queue within
// its link's LQ_UNITS, units exactly when there are Messages, and the non-empty mask holding exactly the non-empty links.
// count[r][s] = the count word of link s -> r (replica indices).
bool link_queues_valid(uint32_t R, uint64_t mask, const uint32_t (*count)[JR_MAX_REPLICAS]) {
  uint64_t want = 0;
  for (uint32_t r = 0; r < R; ++r)
    for (uint32_t s = 0; s < R; ++s) {
      if (s == r) continue;
      const uint32_t c = count[r][s], nm = c & 255u, nu = c >> 8;
      if (nm > JR_LINK_QUEUE_MSGS || nu > LQ_UNITS || (nm == 0) != (nu == 0)) return false;
      if (nm) want |= 1ull << (8 * r + s);
    }
  return mask == want;
}

struct Segment { void* p; size_t n; };
std::vector<Segment> save_segments(jr_engine* e) {
  std::vector<Segment> v;
  for (const PlaneDesc& pd : engine_planes(e)) v.push_back({pd.p, pd.bytes});
  return v;
}
}  // namespace

jr_status jr_engine_save_size(jr_engine* e, size_t* bytes) {
  if (!e || !bytes) return JR_E_INVAL;
  size_t n = sizeof(SaveHeader);
  for (const Segment& sg : save_segments(e)) n += sg.n;
  *bytes = n;
  return JR_OK;
}

jr_status jr_engine_save(jr_engine* e, void* buf, size_t cap) {
  if (!e || !buf) return JR_E_INVAL;
  size_t need = 0;
  jr_engine_save_size(e, &need);
  if (cap < need) return JR_E_CAPACITY;
  CK(cudaSetDevice(e->cfg.device));
  jr_status st = jr_engine_sync(e);
  if (st != JR_OK) return st;
  SaveHeader h;
  memset(&h, 0, sizeof h);
  h.magic = SAVE_MAGIC;
  h.bytes = need;
  h.cfg = e->cfg;
  h.cur = (uint32_t)e->cur;
  h.step_index = e->step_index;
  memcpy(buf, &h, sizeof h);
  char* at = (char*)buf + sizeof h;
  for (const Segment& sg : save_segments(e)) {
    CK(cudaMemcpyAsync(at, sg.p, sg.n, cudaMemcpyDeviceToHost, e->stream));
    at += sg.n;
  }
  CK(cudaStreamSynchronize(e->stream));
  return JR_OK;
}

jr_status jr_engine_restore(jr_engine* e, const void* buf, size_t bytes) {
  if (!e || !buf || bytes < sizeof(SaveHeader)) return JR_E_INVAL;
  SaveHeader h;
  memcpy(&h, buf, sizeof h);
  size_t need = 0;
  jr_engine_save_size(e, &need);
  jr_config a = h.cfg, b = e->cfg;
  a.device = b.device = 0;   // a checkpoint may move to another GPU
  if (h.magic != SAVE_MAGIC || h.bytes != need || bytes < need || memcmp(&a, &b, sizeof a) != 0) {
    set_err("checkpoint does not match this engine's configuration");
    return JR_E_INVAL;
  }
  if (e->d.lq) {   // the link queues, checked before anything reaches the device
    const Dev& d = e->d;
    const unsigned char *qm = nullptr, *qc = nullptr;
    const unsigned char* at = (const unsigned char*)buf + sizeof h;
    for (const Segment& sg : save_segments(e)) {
      if (sg.p == d.lqm) qm = at;
      if (sg.p == d.lqc) qc = at;
      at += sg.n;
    }
    for (uint32_t g = 0; g < d.Gp; ++g) {
      uint64_t m;
      memcpy(&m, qm + 8 * (size_t)g, 8);
      uint32_t count[JR_MAX_REPLICAS][JR_MAX_REPLICAS] = {};
      for (uint32_t r = 0; r < d.R; ++r)
        for (uint32_t s = 0; s < d.R; ++s)
          if (s != r) memcpy(&count[r][s], qc + 4 * (((size_t)lq_slot(r, s) * d.R + r) * d.Gp + g), 4);
      if (!link_queues_valid(d.R, m, count)) {
        set_err("checkpoint: the link queues of group %u are inconsistent or exceed their bounds", g);
        return JR_E_INVAL;
      }
    }
  }
  CK(cudaSetDevice(e->cfg.device));
  jr_status st = jr_engine_sync(e);
  if (st != JR_OK) return st;
  const char* at = (const char*)buf + sizeof h;
  for (const Segment& sg : save_segments(e)) {
    CK(cudaMemcpyAsync(sg.p, at, sg.n, cudaMemcpyHostToDevice, e->stream));
    at += sg.n;
  }
  CK(cudaStreamSynchronize(e->stream));
  e->cur = (int)h.cur;
  e->step_index = h.step_index;
  e->fsm_npending = 0;
  e->resp_b = -1;
  return JR_OK;
}

// ---- group export / import ---------------------------------------------------------------------------------------------
namespace {
struct ImageHeader {
  uint64_t magic;
  uint32_t version, n_groups;
  uint64_t bytes, checksum;      // the whole image; the checksum is taken with this field zero
  jr_config cfg;                 // the source's
  uint32_t rec_units, words;     // fixed record size and the words of its planes: a different plane list is refused
  uint32_t reserved[4];
};
static_assert(sizeof(ImageHeader) % 16 == 0, "the image body starts 16-byte aligned");
constexpr uint64_t IMAGE_MAGIC = 0x4a5247524f555031ull;   // "JRGROUP1"
constexpr uint32_t IMAGE_VERSION = 1;

struct ImgLayout {
  std::vector<ImgPlane> planes;   // the WORDS planes, in list order
  uint32_t words = 0, rec_units = 0;
  uint32_t w_fc = 0, w_tb = 0, w_pnc = ~0u;   // word offsets inside a record's planes
  uint32_t w_lqm = ~0u, w_lqc = ~0u;          // (JR_F_LINK_QUEUES)
};
ImgLayout img_layout(jr_engine* e) {
  ImgLayout L;
  for (const PlaneDesc& pd : engine_planes(e)) {
    if (pd.carry != Carry::WORDS) continue;
    if (pd.p == e->d.fc) L.w_fc = L.words;
    if (pd.p == e->d.tb) L.w_tb = L.words;
    if (pd.p == e->rp.pnc) L.w_pnc = L.words;
    if (pd.p == e->d.lqm) L.w_lqm = L.words;
    if (pd.p == e->d.lqc) L.w_lqc = L.words;
    L.planes.push_back(ImgPlane{(uint32_t*)pd.p, pd.words, pd.depth, pd.per_group ? 1u : 0u});
    L.words += pd.words * pd.depth;
  }
  L.rec_units = 1 + (L.words + 3) / 4;
  return L;
}

// Fields two engines must share for an image of one to run in the other (JR_F_NO_SYMMETRIC_FOLD only picks a code path).
bool image_config_matches(const jr_config& a, const jr_config& b) {
  const uint32_t keep = ~(uint32_t)JR_F_NO_SYMMETRIC_FOLD;
  return a.abi_version == b.abi_version && a.n_replicas == b.n_replicas && a.chain_capacity == b.chain_capacity &&
         a.mailbox_units == b.mailbox_units && a.fsm_units == b.fsm_units && a.election_min_ms == b.election_min_ms &&
         a.election_max_ms == b.election_max_ms && a.heartbeat_ms == b.heartbeat_ms && a.resident_mask == b.resident_mask &&
         (a.flags & keep) == (b.flags & keep);
}

// Four independent multiply-rotate lanes over 8-byte words, folded with mix64: a damaged byte anywhere changes it.
uint64_t image_checksum(const unsigned char* p, size_t n) {
  uint64_t h[4] = {0x243f6a8885a308d3ull, 0x13198a2e03707344ull, 0xa4093822299f31d0ull, 0x082efa98ec4e6c89ull};
  auto lane = [](uint64_t x, uint64_t w) {
    x ^= w * 0x9e3779b97f4a7c15ull;
    return ((x << 31) | (x >> 33)) * 0xbf58476d1ce4e5b9ull;
  };
  size_t k = 0;
  for (; k + 32 <= n; k += 32)
    for (int l = 0; l < 4; ++l) {
      uint64_t w;
      memcpy(&w, p + k + 8 * l, 8);
      h[l] = lane(h[l], w);
    }
  uint64_t tail = 0;
  for (size_t b = 0; k + b < n; ++b) tail = mix64(tail ^ ((uint64_t)p[k + b] << 8 | b));
  return mix64(mix64(mix64(mix64(h[0] ^ n) ^ h[1]) ^ h[2]) ^ h[3] ^ mix64(tail + (n - k)));
}

uint64_t header_checksum(const unsigned char* image, size_t bytes) {
  ImageHeader h;
  memcpy(&h, image, sizeof h);
  h.checksum = 0;
  const uint64_t a = image_checksum(reinterpret_cast<const unsigned char*>(&h), sizeof h);
  return mix64(a ^ image_checksum(image + sizeof h, bytes - sizeof h));
}

inline size_t up16(size_t b) { return (b + 15) / 16 * 16; }
}  // namespace

jr_status jr_group_export(jr_engine* e, const uint32_t* groups, size_t n, void* image, size_t cap, size_t* bytes) {
  if (!e || !bytes || (n && !groups)) return JR_E_INVAL;
  const Dev& d = e->d;
  if (n > d.G) { set_err("more groups than the engine holds"); return JR_E_INVAL; }
  {   // checked before the first device call: on JR_E_INVAL the engine is untouched
    std::vector<uint8_t> seen(d.G, 0);
    for (size_t k = 0; k < n; ++k) {
      if (groups[k] >= d.G || seen[groups[k]]) {
        set_err("groups[%zu]: out of range or named twice", k);
        return JR_E_INVAL;
      }
      seen[groups[k]] = 1;
    }
  }
  CK(cudaSetDevice(e->cfg.device));
  const ImgLayout L = img_layout(e);
  const uint32_t T = CTA_THREADS;
  const size_t reps = (size_t)d.R * n;
  const uint32_t n_ctas = (uint32_t)((reps + T - 1) / T);
  const size_t o_planes = up16(n * sizeof(uint32_t)), o_part = o_planes + up16(L.planes.size() * sizeof(ImgPlane));
  const size_t o_cnt = o_part + up16((size_t)n_ctas * sizeof(unsigned long long));
  jr_status st = scratch_reserve(&e->move_buf, &e->move_cap, o_cnt + reps * sizeof(uint4));
  if (st != JR_OK) return st;
  char* base = (char*)e->move_buf;
  const uint32_t* dgroups = (const uint32_t*)base;
  const ImgPlane* dplanes = (const ImgPlane*)(base + o_planes);
  unsigned long long* dpart = (unsigned long long*)(base + o_part);
  uint4* dcnt = (uint4*)(base + o_cnt);
  const int prev = e->cur ^ 1;   // the mailbox the previous step wrote: the mail in flight
  std::vector<unsigned long long> part(n_ctas);
  if (reps) {
    CK(cudaMemcpyAsync(base, groups, n * sizeof(uint32_t), cudaMemcpyHostToDevice, e->stream));
    CK(cudaMemcpyAsync(base + o_planes, L.planes.data(), L.planes.size() * sizeof(ImgPlane), cudaMemcpyHostToDevice, e->stream));
    JR_LAUNCH(group_count_kernel, n_ctas, T, e->stream, d, dgroups, (uint32_t)n, prev, (const uint32_t*)e->rp.pnc, dcnt, dpart);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(part.data(), dpart, n_ctas * sizeof(unsigned long long), cudaMemcpyDeviceToHost, e->stream));
  }
  CK(cudaStreamSynchronize(e->stream));   // (also covers `groups` and the plane list)
  unsigned long long var = 0;
  for (uint32_t k = 0; k < n_ctas; ++k) { const unsigned long long v = part[k]; part[k] = var; var += v; }
  const size_t body = (reps * L.rec_units + (size_t)var) * sizeof(uint4);
  *bytes = sizeof(ImageHeader) + body;
  if (!image || cap < *bytes) { set_err("the image needs %zu bytes", *bytes); return JR_E_CAPACITY; }
  if (reps) {
    if ((st = scratch_reserve(&e->move_img, &e->move_img_cap, body)) != JR_OK) return st;
    CK(cudaMemcpyAsync(dpart, part.data(), n_ctas * sizeof(unsigned long long), cudaMemcpyHostToDevice, e->stream));
    JR_LAUNCH(group_pack_kernel, n_ctas, T, e->stream, d, dgroups, (uint32_t)n, prev, dplanes, (uint32_t)L.planes.size(),
              L.rec_units, (const uint4*)dcnt, (const unsigned long long*)dpart, (uint4*)e->move_img, e->rp);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync((char*)image + sizeof(ImageHeader), e->move_img, body, cudaMemcpyDeviceToHost, e->stream));
    CK(cudaStreamSynchronize(e->stream));
  }
  ImageHeader h;
  memset(&h, 0, sizeof h);
  h.magic = IMAGE_MAGIC;
  h.version = IMAGE_VERSION;
  h.n_groups = (uint32_t)n;
  h.bytes = *bytes;
  h.cfg = e->cfg;
  h.rec_units = L.rec_units;
  h.words = L.words;
  memcpy(image, &h, sizeof h);
  h.checksum = header_checksum((const unsigned char*)image, *bytes);
  memcpy(image, &h, sizeof h);
  return JR_OK;
}

jr_status jr_group_import(jr_engine* e, const uint32_t* slots, size_t n, const void* image, size_t bytes) {
  if (!e || (n && !slots) || !image) return JR_E_INVAL;
  const Dev& d = e->d;
  // everything is checked before the first device write: on JR_E_INVAL the engine is untouched
  ImageHeader h;
  if (bytes < sizeof h) { set_err("truncated image"); return JR_E_INVAL; }
  memcpy(&h, image, sizeof h);
  const unsigned char* img = (const unsigned char*)image;
  if (h.magic != IMAGE_MAGIC || h.version != IMAGE_VERSION) { set_err("not a group image of this version"); return JR_E_INVAL; }
  if (h.bytes > bytes || h.bytes < sizeof h) { set_err("truncated image"); return JR_E_INVAL; }
  if (header_checksum(img, h.bytes) != h.checksum) { set_err("image checksum mismatch"); return JR_E_INVAL; }
  if (h.n_groups != n) { set_err("the image holds %u groups, %zu slots given", h.n_groups, n); return JR_E_INVAL; }
  {
    std::vector<uint8_t> seen(d.G, 0);
    for (size_t k = 0; k < n; ++k) {
      if (slots[k] >= d.G || seen[slots[k]]) {
        set_err("slots[%zu]: out of range or named twice", k);
        return JR_E_INVAL;
      }
      seen[slots[k]] = 1;
    }
  }
  if (!image_config_matches(h.cfg, e->cfg)) { set_err("the image's engine configuration does not match this engine's"); return JR_E_INVAL; }
  const ImgLayout L = img_layout(e);
  if (h.rec_units != L.rec_units || h.words != L.words) { set_err("the image's record layout does not match"); return JR_E_INVAL; }
  const size_t reps = (size_t)d.R * n, fixed = reps * L.rec_units;
  const size_t body = (size_t)h.bytes - sizeof h;
  if (body % sizeof(uint4) || body / sizeof(uint4) < fixed) { set_err("truncated image"); return JR_E_INVAL; }
  const size_t units = body / sizeof(uint4);
  auto unit = [&](size_t u) { uint4 v; memcpy(&v, img + sizeof h + u * sizeof(uint4), sizeof v); return v; };
  auto word = [&](size_t t, uint32_t w) { uint32_t v; memcpy(&v, img + sizeof h + (t * L.rec_units + 1) * sizeof(uint4) + 4 * (size_t)w, 4); return v; };
  std::vector<unsigned long long> off(reps);
  std::vector<uint32_t> floor(n);
  unsigned long long at = 0;
  for (size_t t = 0; t < reps; ++t) {   // counts, first
    const size_t j = t % n;
    const uint4 c = unit(t * L.rec_units);
    const uint32_t fcx = word(t, L.w_fc), fl = word(t, L.w_tb);
    const bool capture = (d.flags & JR_F_CAPTURE_FSM) != 0;
    if (c.x > d.cap || c.y > d.U || c.z > (capture ? d.F : 0u) || c.z != std::min(fcx, capture ? d.F : 0u) ||
        c.w > (e->rp.pn ? JR_NOTIFY_RUNS : 0u) || (L.w_pnc != ~0u && word(t, L.w_pnc) != c.w)) {
      set_err("record %zu: counts outside the engine's limits", t);
      return JR_E_INVAL;
    }
    if (t < n) floor[j] = fl;
    if (fl >= JR_BLOCK_ID_LIMIT || fl != floor[j]) { set_err("record %zu: floor >= 2^31 or not the group's", t); return JR_E_INVAL; }
    off[t] = at;
    at += (unsigned long long)c.x + c.y + 2ull * c.z + 2ull * c.w;
  }
  if (fixed + at != units) { set_err("truncated image"); return JR_E_INVAL; }
  if (L.w_lqm != ~0u)   // the link queues: each group's mask (carried in its first replica's record) against its counts
    for (size_t j = 0; j < n; ++j) {
      const uint64_t m = (uint64_t)word(j, L.w_lqm) | ((uint64_t)word(j, L.w_lqm + 1) << 32);
      uint32_t count[JR_MAX_REPLICAS][JR_MAX_REPLICAS] = {};
      for (uint32_t r = 0; r < d.R; ++r)
        for (uint32_t s = 0; s < d.R; ++s)
          if (s != r) count[r][s] = word((size_t)r * n + j, L.w_lqc + lq_slot(r, s));
      if (!link_queues_valid(d.R, m, count)) {
        set_err("group %zu of the image: link queues inconsistent or beyond their bounds", j);
        return JR_E_INVAL;
      }
    }
  for (size_t t = 0; t < reps; ++t) {   // then the rows: ascending, inside the window, below 2^31 (D4, D7)
    const uint32_t rows = unit(t * L.rec_units).x;
    const uint64_t lo = floor[t % n];
    for (uint32_t k = 0; k < rows; ++k) {
      const uint4 b = unit(fixed + off[t] + k);
      if (b.x < lo || b.x - lo >= d.cap || b.x >= JR_BLOCK_ID_LIMIT || b.y >= JR_BLOCK_ID_LIMIT ||
          (k && b.x <= unit(fixed + off[t] + k - 1).x)) {
        set_err("record %zu row %u: id not ascending, outside [floor, floor + chain_capacity) or >= 2^31, or next >= 2^31", t, k);
        return JR_E_INVAL;
      }
    }
  }
  if (n == 0) return JR_OK;
  CK(cudaSetDevice(e->cfg.device));
  const size_t o_planes = up16(n * sizeof(uint32_t)), o_off = o_planes + up16(L.planes.size() * sizeof(ImgPlane));
  jr_status st = scratch_reserve(&e->move_buf, &e->move_cap, o_off + reps * sizeof(unsigned long long));
  if (st != JR_OK) return st;
  if ((st = scratch_reserve(&e->move_img, &e->move_img_cap, body)) != JR_OK) return st;
  char* base = (char*)e->move_buf;
  CK(cudaMemcpyAsync(base, slots, n * sizeof(uint32_t), cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemcpyAsync(base + o_planes, L.planes.data(), L.planes.size() * sizeof(ImgPlane), cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemcpyAsync(base + o_off, off.data(), reps * sizeof(unsigned long long), cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemcpyAsync(e->move_img, img + sizeof h, body, cudaMemcpyHostToDevice, e->stream));
  JR_LAUNCH(group_unpack_kernel, (unsigned)((n + 127) / 128), 128, e->stream, d, (const uint32_t*)base, (uint32_t)n, e->cur ^ 1,
            (const ImgPlane*)(base + o_planes), (uint32_t)L.planes.size(), L.rec_units, (const uint4*)e->move_img,
            (const unsigned long long*)(base + o_off), e->rp);
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(e->stream));
  return JR_OK;
}

jr_status jr_set_alive(jr_engine* e, uint32_t group, uint32_t node, int alive) {
  if (!e || group >= e->d.G || node < 1 || node > e->d.R) return JR_E_INVAL;
  CK(cudaSetDevice(e->cfg.device));
  JR_LAUNCH(set_alive_kernel, 1, 1, e->stream, e->d, group, node - 1, alive);
  CK(cudaGetLastError());
  return JR_OK;
}

jr_status jr_kill_leaders(jr_engine* e, uint64_t salt, uint32_t permille, uint64_t* n_killed) {
  if (!e) return JR_E_INVAL;
  CK(cudaSetDevice(e->cfg.device));
  CK(cudaMemsetAsync(e->scratch, 0, sizeof(unsigned long long), e->stream));
  JR_LAUNCH(kill_leaders_kernel, (e->d.G + 127) / 128, 128, e->stream, e->d, mix64(e->d.seed ^ salt), permille, e->scratch);
  CK(cudaGetLastError());
  uint64_t k = 0;
  CK(cudaMemcpyAsync(&k, e->scratch, sizeof k, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  if (n_killed) *n_killed = k;
  return JR_OK;
}

// ---- peer links (JR_F_PEER_LINKS) ------------------------------------------------------------------------------------
// The bits a link matrix of an R-replica group may hold: 8*(r-1) + (s-1) for receivers and senders 1..R, r != s.
static uint64_t links_valid_mask(uint32_t R) {
  uint64_t m = 0;
  for (uint32_t r = 0; r < R; ++r) m |= (((1ull << R) - 1ull) & ~(1ull << r)) << (8u * r);
  return m;
}

// groups == NULL: n must be G (dense).  Otherwise every group in range and named once.  Checked on the host first.
static jr_status links_check_groups(jr_engine* e, const uint32_t* groups, size_t n, const char* what) {
  if (!e->d.links) { set_err("%s: engine created without JR_F_PEER_LINKS", what); return JR_E_INVAL; }
  if (!groups) {
    if (n != e->d.G) { set_err("%s: groups == NULL needs n == n_groups", what); return JR_E_INVAL; }
    return JR_OK;
  }
  if (n > e->d.G) { set_err("%s: more groups than the engine holds", what); return JR_E_INVAL; }
  std::vector<uint8_t> seen(e->d.G, 0);
  for (size_t k = 0; k < n; ++k) {
    if (groups[k] >= e->d.G || seen[groups[k]]) { set_err("%s: groups[%zu] out of range or named twice", what, k); return JR_E_INVAL; }
    seen[groups[k]] = 1;
  }
  return JR_OK;
}

jr_status jr_set_links(jr_engine* e, const uint32_t* groups, const uint64_t* cuts, size_t n) {
  if (!e || (n && !cuts)) return JR_E_INVAL;
  jr_status st = links_check_groups(e, groups, n, "jr_set_links");
  if (st != JR_OK) return st;
  const uint64_t bad = ~links_valid_mask(e->d.R);
  for (size_t k = 0; k < n; ++k)
    if (cuts[k] & bad) { set_err("jr_set_links: cuts[%zu] has a bit on the diagonal or above n_replicas", k); return JR_E_INVAL; }
  if (n == 0) return JR_OK;
  CK(cudaSetDevice(e->cfg.device));
  if (!groups) {
    CK(cudaMemcpyAsync(e->d.links, cuts, n * sizeof(uint64_t), cudaMemcpyHostToDevice, e->stream));
  } else {   // one copy: {cuts, groups}, then the scatter
    std::vector<unsigned char> in(n * (sizeof(uint64_t) + sizeof(uint32_t)));
    memcpy(in.data(), cuts, n * sizeof(uint64_t));
    memcpy(in.data() + n * sizeof(uint64_t), groups, n * sizeof(uint32_t));
    if ((st = many_reserve(e, in.size())) != JR_OK) return st;
    CK(cudaMemcpyAsync(e->many_buf, in.data(), in.size(), cudaMemcpyHostToDevice, e->stream));
    JR_LAUNCH(links_scatter_kernel, (unsigned)((n + 127) / 128), 128, e->stream, e->d, (const unsigned long long*)e->many_buf,
              (const uint32_t*)((char*)e->many_buf + n * sizeof(uint64_t)), (uint32_t)n);
    CK(cudaGetLastError());
  }
  CK(cudaStreamSynchronize(e->stream));
  return JR_OK;
}

jr_status jr_get_links(jr_engine* e, const uint32_t* groups, size_t n, uint64_t* out) {
  if (!e || (n && !out)) return JR_E_INVAL;
  jr_status st = links_check_groups(e, groups, n, "jr_get_links");
  if (st != JR_OK) return st;
  if (n == 0) return JR_OK;
  CK(cudaSetDevice(e->cfg.device));
  if (!groups) {
    CK(cudaMemcpyAsync(out, e->d.links, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, e->stream));
  } else {   // the group list in, the gather, the matrices out
    if ((st = many_reserve(e, n * (sizeof(uint64_t) + sizeof(uint32_t)))) != JR_OK) return st;
    unsigned long long* dout = (unsigned long long*)e->many_buf;
    uint32_t* dgroups = (uint32_t*)(dout + n);
    CK(cudaMemcpyAsync(dgroups, groups, n * sizeof(uint32_t), cudaMemcpyHostToDevice, e->stream));
    JR_LAUNCH(links_gather_kernel, (unsigned)((n + 127) / 128), 128, e->stream, e->d, (const uint32_t*)dgroups, (uint32_t)n, dout);
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(out, dout, n * sizeof(uint64_t), cudaMemcpyDeviceToHost, e->stream));
  }
  CK(cudaStreamSynchronize(e->stream));
  return JR_OK;
}

jr_status jr_get_link_queues(jr_engine* e, const uint32_t* groups, size_t n, uint8_t* depths) {
  if (!e || (n && !depths)) return JR_E_INVAL;
  if (!e->d.lq) { set_err("jr_get_link_queues: engine created without JR_F_LINK_QUEUES"); return JR_E_INVAL; }
  jr_status st = links_check_groups(e, groups, n, "jr_get_link_queues");
  if (st != JR_OK) return st;
  if (n == 0) return JR_OK;
  CK(cudaSetDevice(e->cfg.device));
  const size_t o_grp = n * 64;   // the depths, then the group list
  if ((st = many_reserve(e, o_grp + (groups ? n * sizeof(uint32_t) : 0))) != JR_OK) return st;
  uint8_t* dout = (uint8_t*)e->many_buf;
  uint32_t* dgroups = groups ? (uint32_t*)(dout + o_grp) : nullptr;
  if (groups) CK(cudaMemcpyAsync(dgroups, groups, n * sizeof(uint32_t), cudaMemcpyHostToDevice, e->stream));
  JR_LAUNCH(link_queues_gather_kernel, (unsigned)((n + 127) / 128), 128, e->stream, e->d, (const uint32_t*)dgroups, (uint32_t)n, dout);
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(depths, dout, n * 64, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return JR_OK;
}

jr_status jr_isolate_leaders(jr_engine* e, uint64_t salt, uint32_t permille, uint64_t* n_isolated) {
  if (!e) return JR_E_INVAL;
  if (!e->d.links) { set_err("jr_isolate_leaders: engine created without JR_F_PEER_LINKS"); return JR_E_INVAL; }
  CK(cudaSetDevice(e->cfg.device));
  CK(cudaMemsetAsync(e->scratch, 0, sizeof(unsigned long long), e->stream));
  JR_LAUNCH(isolate_leaders_kernel, (e->d.G + 127) / 128, 128, e->stream, e->d, mix64(e->d.seed ^ salt), permille, e->scratch);
  CK(cudaGetLastError());
  uint64_t k = 0;
  CK(cudaMemcpyAsync(&k, e->scratch, sizeof k, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  if (n_isolated) *n_isolated = k;
  return JR_OK;
}

jr_status jr_leader_table_device(jr_engine* e, void* dev_out) {
  if (!e || !dev_out) return JR_E_INVAL;
  CK(cudaSetDevice(e->cfg.device));
  JR_LAUNCH(leader_table_kernel, (e->d.G + 127) / 128, 128, e->stream, e->d, (jr_leader_entry*)dev_out, e->route);
  CK(cudaGetLastError());
  return JR_OK;
}

jr_status jr_leader_table_async(jr_engine* e, jr_leader_entry* host_out) {
  if (!e || !host_out) return JR_E_INVAL;
  const int b = e->tab_i;
  e->tab_i = (b + 1) % jr_engine::NBUF;
  if (e->tab_used[b]) CK(cudaStreamWaitEvent(e->stream, e->tab_free[b], 0));  // its last copy-out is done
  jr_status st = jr_leader_table_device(e, e->leaders[b]);
  if (st != JR_OK) return st;
  CK(cudaEventRecord(e->tab_ready[b], e->stream));
  CK(cudaStreamWaitEvent(e->d2h, e->tab_ready[b], 0));
  CK(cudaMemcpyAsync(host_out, e->leaders[b], (size_t)e->d.G * sizeof(jr_leader_entry), cudaMemcpyDeviceToHost, e->d2h));
  CK(cudaEventRecord(e->tab_free[b], e->d2h));
  e->tab_used[b] = true;
  std::lock_guard<std::mutex> l(e->qmu);
  if (e->tab_npending == jr_engine::NBUF) {  // the oldest one is about to be overwritten anyway
    for (int k = 0; k + 1 < jr_engine::NBUF; ++k) e->tab_pending[k] = e->tab_pending[k + 1];
    --e->tab_npending;
  }
  e->tab_pending[e->tab_npending++] = b;
  return JR_OK;
}

jr_status jr_leader_table_wait(jr_engine* e) {
  if (!e) return JR_E_INVAL;
  CK(cudaSetDevice(e->cfg.device));
  int b;
  {
    std::lock_guard<std::mutex> l(e->qmu);
    if (e->tab_npending == 0) return JR_OK;
    b = e->tab_pending[0];
    for (int k = 0; k + 1 < jr_engine::NBUF; ++k) e->tab_pending[k] = e->tab_pending[k + 1];
    --e->tab_npending;
  }
  CK(cudaEventSynchronize(e->tab_free[b]));
  return JR_OK;
}

jr_status jr_leader_table(jr_engine* e, jr_leader_entry* host_out) {
  jr_status st = jr_leader_table_async(e, host_out);
  if (st != JR_OK) return st;
  CK(cudaStreamSynchronize(e->d2h));
  std::lock_guard<std::mutex> l(e->qmu);   // a consumer thread may sit in jr_leader_table_wait
  e->tab_npending = 0;
  return JR_OK;
}

}  // extern "C"
