// Sliding-band pull wavefront engine (sm_90a).
//
// What it replaces: the heap loops of the reference
//   CVPMeshPlanner::waveFrontPropagation   cvp_mesh_planner.cpp:747-886
//   DijkstraMeshPlanner::dijkstra          dijkstra_mesh_planner.cpp:287-348
//   InflationLayer::waveCostInflation      inflation_layer.cpp:407-478
// which pop one vertex at a time from lvr2::Meap and push updates to the free
// vertex of every incident face (edge) that has all its other vertices fixed.
//
// GPU formulation (not a translation of the heap):
//   * every vertex carries one 16-byte word  {d : potential, a1, a2, a3 : pop time}.
//     The pop time is the moment the sequential algorithm would have popped the
//     vertex, as a monotonic stack of water levels (problems.cuh); for causal
//     updates it is simply (d, id)  ==  the oracle's canonical heap order.
//   * a *candidate* vertex is recomputed FROM SCRATCH ("pull") from its corner
//     records: the faces are visited in the order their later source vertex
//     pops, and a face only fires while the candidate itself has not popped yet.
//     That vertex-local replay reproduces the sequential result including the
//     non-causal "back-steps" of the CVP unfolding update (SURVEY.md H1); the
//     CPU simulator of exactly this rule is bit-identical to the oracle on the
//     10k / 1M meshes, and these very sources run on a CPU interpreter in the test-suite (tests/emu).
//   * candidates within a sliding band [lo, lo+delta) of potentials are
//     recomputed every round; everything whose tau lies strictly below the
//     smallest tau that changed in the round is a converged prefix and leaves
//     the list ("settled").  One barrier per round.
//   * one wavefront is owned by ONE thread-block cluster (CS CTAs, CS in
//     {1,2,4,8,16}); the barrier is the hardware cluster barrier (or
//     __syncthreads for CS==1), not a grid-wide sync, so a round costs ~1 us
//     instead of a kernel launch.  Batches run one wavefront per cluster on all
//     SMs; CS==0 selects a cooperative whole-grid group (used by the
//     multi-source inflation wave which has few, very wide rounds).
//   * the next round's candidate list is staged in shared memory per CTA and
//     flushed with one global atomic per CTA per round.
#pragma once
#include <cooperative_groups.h>
#include <cstdint>

#include "wavefront_math.cuh"

namespace mnb {
namespace cg = cooperative_groups;

constexpr uint32_t INF_BITS = 0x7f800000u;
constexpr int STAGNATION_ROUNDS = 24;

// Pop time of a vertex = the moment the sequential algorithm pops it, written as the stack of canonical heap keys
// (key, vertex id) that were running maxima of the pop sequence at that moment ("water levels"):
//     L1 > L2 > ... > Ln,   Ln = the vertex's own (key, id).
// A vertex that pops at its own key has n = 1 (the oracle's canonical heap order).  A non-causal "back-step" label
// (X, c) <= the pop time F of the face that hands it out is popped inside the cascade that runs below the water line:
// it keeps the levels of F that are > (X, c) and appends (X, c) (problems.cuh, TimeAlg::accept).  Times compare
// lexicographically, a proper prefix first (a trigger pops before the members of its cascade).  Cascades nest to any
// depth; the representation is exact for all of them:
//   * levels 1-3 keys live in the 16-byte label word {d, a1, a2, a3} (0 = level absent; pop keys are > 0 below level 1);
//   * the id of level 1 ("root") lives in a side array when it differs from the vertex (sign bit of the a2 word);
//   * n == 3: the id of level 2 is the side word `ext`;  n >= 4: ext = EXT_POOL | offset of a record
//     [n, id2, id3, key4, id4, ..., keyn, idn] in the per-wavefront level pool (sign bit of the a3 word = "ext valid").
// float32 potentials collide millions of times on 10M-vertex meshes, hence the ids at every level: without them a
// cascade under a tied key was ordered after ALL plain labels of that key.
constexpr uint32_t EXT_POOL = 0x80000000u;
struct EvTime { float a1, a2, a3; uint32_t root, ext, self; };
__device__ __forceinline__ EvTime ev_normal(float key, uint32_t id) { EvTime t; t.a1 = key; t.a2 = 0.0f; t.a3 = 0.0f; t.root = id; t.ext = 0u; t.self = id; return t; }
// per-vertex label: one 16-byte word {d, a1, a2 | root flag, a3 | ext flag}
struct Label { float d; EvTime t; };
__device__ __forceinline__ uint4 state_inf() { return make_uint4(INF_BITS, INF_BITS, 0u, 0u); }

// Comparison of pop times.  `pool` is the level pool of the wavefront (only dereferenced when two times tie through a
// level whose id or key lives there -- never on the hot path).
struct TimeAlg {
  const uint32_t* pool = nullptr;
  __device__ __forceinline__ uint32_t id2_of(const EvTime& t) const {      // id of level 2 (level 2 must exist)
    return t.a3 == 0.0f ? t.self : ((t.ext & EXT_POOL) ? __ldcg(&pool[(t.ext & ~EXT_POOL) + 1]) : t.ext);
  }
  __device__ __forceinline__ uint32_t id3_of(const EvTime& t) const {      // id of level 3 (level 3 must exist)
    return (t.ext & EXT_POOL) ? __ldcg(&pool[(t.ext & ~EXT_POOL) + 2]) : t.self;
  }
  __device__ __forceinline__ uint32_t levels_of(const EvTime& t) const {
    return t.a2 == 0.0f ? 1u : (t.a3 == 0.0f ? 2u : ((t.ext & EXT_POOL) ? __ldcg(&pool[t.ext & ~EXT_POOL]) : 3u));
  }
  // levels 2.. tie on the key of level 2 (rare: same cascade, bit-identical keys or the same sub-trigger)
  // (the out-of-line helpers take pop times BY VALUE: a by-reference argument of a __noinline__ callee forces the caller's
  // variable into local memory for its whole lifetime -- labels a, b, T and tc of the hot path were stored to the stack on
  // every evaluation while these took references)
  __device__ __noinline__ bool less_tail(const EvTime x, const EvTime y) const {
    const uint32_t i2x = id2_of(x), i2y = id2_of(y);
    if (i2x != i2y) return i2x < i2y;
    if (x.a3 != y.a3) return x.a3 < y.a3;
    if (x.a3 == 0.0f) return false;                                 // the same vertex
    const uint32_t i3x = id3_of(x), i3y = id3_of(y);
    if (i3x != i3y) return i3x < i3y;
    const uint32_t nx = levels_of(x), ny = levels_of(y);
    const uint32_t ox = x.ext & ~EXT_POOL, oy = y.ext & ~EXT_POOL;
    for (uint32_t i = 4;; ++i) {
      if (i > nx) return i <= ny;                                   // x is a prefix of y (or the same time)
      if (i > ny) return false;
      const uint32_t kx = __ldcg(&pool[ox + 3 + 2 * (i - 4)]), ky = __ldcg(&pool[oy + 3 + 2 * (i - 4)]);
      if (kx != ky) return kx < ky;                                 // keys are > 0: bit order = value order
      const uint32_t ix = __ldcg(&pool[ox + 4 + 2 * (i - 4)]), iy = __ldcg(&pool[oy + 4 + 2 * (i - 4)]);
      if (ix != iy) return ix < iy;
    }
  }
  __device__ __forceinline__ bool tless(const EvTime& x, const EvTime& y) const {
    if (x.a1 != y.a1) return x.a1 < y.a1;
    if (x.root != y.root) return x.root < y.root;
    if (x.a2 != y.a2) return x.a2 < y.a2;                           // 0 = no level 2: a prefix sorts first
    if (x.a2 == 0.0f) return false;                                 // both are the vertex (a1, root) itself
    return less_tail(x, y);
  }
  __device__ __noinline__ bool eq_pool(const EvTime x, const EvTime y) const {
    if (!(x.ext & y.ext & EXT_POOL)) return false;
    const uint32_t ox = x.ext & ~EXT_POOL, oy = y.ext & ~EXT_POOL;
    if (ox == oy) return true;
    const uint32_t n = __ldcg(&pool[ox]);
    if (n != __ldcg(&pool[oy])) return false;
    for (uint32_t i = 1; i < 3 + 2 * (n - 3); ++i) if (__ldcg(&pool[ox + i]) != __ldcg(&pool[oy + i])) return false;
    return true;
  }
  __device__ __forceinline__ bool teq(const EvTime& x, const EvTime& y) const {
    if (__float_as_uint(x.a1) != __float_as_uint(y.a1) || __float_as_uint(x.a2) != __float_as_uint(y.a2) ||
        __float_as_uint(x.a3) != __float_as_uint(y.a3) || x.root != y.root || x.self != y.self) return false;
    if ((x.ext | y.ext) & EXT_POOL) return eq_pool(x, y);
    return x.ext == y.ext;
  }
};

// A pop time under construction (the serial replays of problems.cuh): either a plain EvTime (n <= 3: `t` is complete) or,
// for n >= 4, a VIRTUAL stack -- levels 1-3 in t.{a1,root,a2,a3} + id2/id3, levels 4..n-1 taken from the pool record
// `src` of the trigger it was derived from, level n = (last, t.self).  Only a label that really changed is written to
// the pool (LabelStore::finish), so recomputing a deep label over and over allocates nothing.
struct EvFull { EvTime t; uint32_t id2, id3, n, src; float last; };

// Labels in global memory + the level pool (shared by the CVP and inflation problems)
struct LabelStore : TimeAlg {
  uint4* state;                         // {d bits, a1 bits, a2 bits | root flag, a3 bits | ext flag}
  uint32_t* root_arr;                   // id of level 1 where it differs from the vertex (cascade members)
  uint32_t* ext_arr;                    // n == 3: id of level 2;  n >= 4: EXT_POOL | pool offset
  uint32_t* chg;                        // 1 + round of the last RE-label of a vertex (0 = never)
  uint32_t* pool_w;                     // == pool (writable)
  unsigned int* pool_top; unsigned int* pool_overflow; uint32_t pool_cap;

  // decoding of the 16-byte label word: sign bit of .z = "level-1 id differs from the vertex, see root_arr",
  // sign bit of .w = "ext_arr valid" (pop-time levels are >= 0, so both bits are free)
  __device__ __forceinline__ Label unpack_label(uint32_t v, const uint4& s) const {
    Label l; l.d = __uint_as_float(s.x); l.t.a1 = __uint_as_float(s.y); l.t.a2 = __uint_as_float(s.z & 0x7fffffffu);
    l.t.a3 = __uint_as_float(s.w & 0x7fffffffu);
    l.t.root = (s.z >> 31) ? __ldcg(&root_arr[v]) : v;
    l.t.ext = (s.w >> 31) ? __ldcg(&ext_arr[v]) : 0u;
    l.t.self = v;
    return l;
  }
  __device__ __forceinline__ Label load_label(uint32_t v) const { return unpack_label(v, __ldcg(&state[v])); }
  // the 16-byte word of a label as store_label() writes it
  __device__ __forceinline__ uint4 pack_label(uint32_t c, float d, const EvTime& t) const {
    uint32_t z = __float_as_uint(t.a2), w = __float_as_uint(t.a3);
    if (t.root != c) z |= 0x80000000u;
    if (t.a3 != 0.0f) w |= 0x80000000u;
    return make_uint4(__float_as_uint(d), __float_as_uint(t.a1), z, w);
  }
  __device__ __forceinline__ void store_label(uint32_t c, float d, const EvTime& t, bool relabel, uint32_t round) const {
    if (t.root != c) __stcg(&root_arr[c], t.root);
    if (t.a3 != 0.0f) __stcg(&ext_arr[c], t.ext);
    if (relabel) __stcg(&chg[c], round + 1u);
    __stcg(&state[c], pack_label(c, d, t));
  }

  // (key bits, id) of level i of a materialised time
  __device__ __forceinline__ void level_of(const EvTime& T, uint32_t i, uint32_t& kb, uint32_t& id) const {
    if (i == 1) { kb = __float_as_uint(T.a1); id = T.root; }
    else if (i == 2) { kb = __float_as_uint(T.a2); id = id2_of(T); }
    else if (i == 3) { kb = __float_as_uint(T.a3); id = id3_of(T); }
    else { const uint32_t o = (T.ext & ~EXT_POOL) + 3 + 2 * (i - 4); kb = __ldcg(&pool[o]); id = __ldcg(&pool[o + 1]); }
  }
  // Does the stack of T hold a level of vertex c?  Then T pops inside a cascade that c started, i.e. AFTER c: a face with
  // that pop time cannot update c.  In a consistent state the time comparison says the same; while labels are still
  // moving, T may rest on a former label of c (a "ghost" level), and accepting its back-step would let c and T support
  // each other -- a stable fixed point of the pull iteration that the sequential order does not have (found by the
  // randomised tests as soon as the stacks were exact).  Such a face does not fire; T itself is re-evaluated because its
  // source c changed.
  __device__ __noinline__ bool names_slow(const EvTime T, uint32_t c) const {
    if (T.root == c || id2_of(T) == c) return true;
    if (T.a3 == 0.0f) return false;
    if (id3_of(T) == c) return true;
    const uint32_t n = levels_of(T);
    for (uint32_t i = 4; i <= n; ++i) { uint32_t kb, id; level_of(T, i, kb, id); if (id == c) return true; }
    return false;
  }
  __device__ __forceinline__ bool names(const EvTime& T, uint32_t c) const { return T.a2 != 0.0f && names_slow(T, c); }
  // One accepted update with value X from a face that fired at time F: c enters the heap with key (X, c) at that moment
  // and pops once everything smaller has popped -- its pop time keeps the levels of F that are > (X, c) and appends (X, c).
  // X == F.a1 exactly: c pops in (key, id) order among the vertices of that key that are still queued -- as a plain label
  // if its id is above the root's, else inside the cascade.
  // Lean form: returns false (t untouched) if the result needs more than 3 levels.
  __device__ __forceinline__ bool accept_lean(uint32_t c, float X, const EvTime& F, EvTime& t) const {
    if (X > F.a1 || (X == F.a1 && c > F.root)) { t = ev_normal(X, c); return true; }        // above water: pops at its own key
    if (F.a2 == 0.0f) { t = F; t.a2 = X; t.self = c; t.ext = 0u; return true; }             // first level of F's cascade
    const uint32_t i2 = id2_of(F);
    if (X > F.a2 || (X == F.a2 && c > i2)) { t.a1 = F.a1; t.root = F.root; t.a2 = X; t.a3 = 0.0f; t.ext = 0u; t.self = c; return true; }
    if (F.a3 != 0.0f) {
      const uint32_t i3 = id3_of(F);
      if (!(X > F.a3 || (X == F.a3 && c > i3))) return false;                               // a fourth level (or more)
    }
    t.a1 = F.a1; t.root = F.root; t.a2 = F.a2; t.a3 = X; t.ext = i2; t.self = c;
    return true;
  }
  __device__ __noinline__ void accept_deep(uint32_t c, float X, const EvTime F, EvFull& o) const {
    const uint32_t nF = levels_of(F), xb = __float_as_uint(X);
    uint32_t k = 3;                                     // (accept_lean has established that levels 1-3 of F stay)
    for (uint32_t i = 4; i <= nF; ++i) {
      uint32_t kb, id; level_of(F, i, kb, id);
      if (kb > xb || (kb == xb && id > c)) k = i; else break;
    }
    o.t.a1 = F.a1; o.t.root = F.root; o.t.a2 = F.a2; o.t.a3 = F.a3; o.t.ext = 0u; o.t.self = c;
    o.id2 = id2_of(F); o.id3 = id3_of(F); o.n = k + 1; o.src = F.ext & ~EXT_POOL; o.last = X;
  }
  __device__ __forceinline__ void accept(uint32_t c, float X, const EvTime& F, EvFull& o) const {
    if (accept_lean(c, X, F, o.t)) o.n = 1u;            // (any value <= 3: `t` is complete)
    else accept_deep(c, X, F, o);
  }
  __device__ __forceinline__ static EvFull full_normal(float key, uint32_t c) { EvFull f; f.t = ev_normal(key, c); f.id2 = c; f.id3 = c; f.n = 1u; f.src = 0u; f.last = 0.0f; return f; }
  // (key bits, id) of level i >= 4 of a virtual time
  __device__ __forceinline__ void vlevel_of(const EvFull& x, uint32_t i, uint32_t& kb, uint32_t& id) const {
    if (i == x.n) { kb = __float_as_uint(x.last); id = x.t.self; }
    else { const uint32_t o = x.src + 3 + 2 * (i - 4); kb = __ldcg(&pool[o]); id = __ldcg(&pool[o + 1]); }
  }
  __device__ __noinline__ bool less_T_deep(const EvTime T, const EvFull& x) const {
    if (T.a1 != x.t.a1) return T.a1 < x.t.a1;
    if (T.root != x.t.root) return T.root < x.t.root;
    if (T.a2 == 0.0f) return true;                      // T is a proper prefix of x
    if (T.a2 != x.t.a2) return T.a2 < x.t.a2;
    const uint32_t i2 = id2_of(T);
    if (i2 != x.id2) return i2 < x.id2;
    if (T.a3 == 0.0f) return true;
    if (T.a3 != x.t.a3) return T.a3 < x.t.a3;
    const uint32_t i3 = id3_of(T);
    if (i3 != x.id3) return i3 < x.id3;
    const uint32_t nT = levels_of(T);
    for (uint32_t i = 4;; ++i) {
      if (i > x.n) return false;                        // x ended: x is a prefix of T (or the same time)
      if (i > nT) return true;
      uint32_t kt, it, kx, ixx; level_of(T, i, kt, it); vlevel_of(x, i, kx, ixx);
      if (kt != kx) return kt < kx;
      if (it != ixx) return it < ixx;
    }
  }
  // is the materialised time T earlier than the time x under construction?
  __device__ __forceinline__ bool less_T_full(const EvTime& T, const EvFull& x) const {
    return x.n <= 3u ? tless(T, x.t) : less_T_deep(T, x);
  }
  __device__ __noinline__ bool eq_deep(const EvFull& x, const EvTime T) const {
    if (__float_as_uint(T.a1) != __float_as_uint(x.t.a1) || __float_as_uint(T.a2) != __float_as_uint(x.t.a2) ||
        __float_as_uint(T.a3) != __float_as_uint(x.t.a3) || T.root != x.t.root || T.self != x.t.self || !(T.ext & EXT_POOL)) return false;
    if (levels_of(T) != x.n || id2_of(T) != x.id2 || id3_of(T) != x.id3) return false;
    for (uint32_t i = 4; i <= x.n; ++i) {
      uint32_t kt, it, kx, ixx; level_of(T, i, kt, it); vlevel_of(x, i, kx, ixx);
      if (kt != kx || it != ixx) return false;
    }
    return true;
  }
  __device__ __noinline__ EvTime materialise(const EvFull& x) const {
    EvTime t = x.t;
    const uint32_t need = 3u + 2u * (x.n - 3u);
    const uint32_t off = atomicAdd(pool_top, need);
    if (off + need > pool_cap || off + need < off) {    // pool exhausted: reported by the host as an error (no silent inexact result)
      *pool_overflow = 1u;
      t.ext = x.id2;                                    // (a well-formed 3-level time so that the wave still terminates)
      return t;
    }
    pool_w[off] = x.n; pool_w[off + 1] = x.id2; pool_w[off + 2] = x.id3;
    for (uint32_t i = 4; i <= x.n; ++i) { uint32_t kb, id; vlevel_of(x, i, kb, id); pool_w[off + 3 + 2 * (i - 4)] = kb; pool_w[off + 4 + 2 * (i - 4)] = id; }
    __threadfence();                                    // the record before the label word that points to it
    t.ext = EXT_POOL | off;
    return t;
  }
  // the label time to store for c: the old one if nothing changed (no allocation), a fresh pool record otherwise
  __device__ __forceinline__ EvTime finish(const EvFull& x, const EvTime& old_t) const {
    if (x.n <= 3u) return x.t;
    if (eq_deep(x, old_t)) return old_t;
    return materialise(x);
  }
};

// mark[] values
constexpr uint32_t MARK_NONE = 0, MARK_CAND = 1, MARK_FIXED = 2, MARK_CAND_ACT = 3;

struct GroupCtl {               // one per wavefront group, global memory
  unsigned int count[3];        // candidate list sizes (ring over rounds)
  unsigned int m_tau[3];        // float bits: min tau touched by a change in the round
  unsigned int lo[3];           // float bits: min pop time over surviving candidates
  // goal_dist (cvp:738,769 / dijkstra:279,296) and the cancel flag are read by EVERY thread at the
  // top of a round and decide whether the group leaves the loop, so they must not change while a
  // round is running: round r reads slot r&1, writers of round r only touch slot (r+1)&1.
  unsigned int goal_ring[2];    // float bits, monotonically decreasing (atomicMin)
  unsigned int stop_ring[2];
  unsigned int goal_bits;       // final goal_dist, published after the last round
  // pop time of the vertex that armed the cutoff (a1 bits, root, a2 bits, a3 bits, ext, vertex): a vertex beyond goal_dist that
  // popped BEFORE that moment did expand in the reference (cvp:754 tests the goal_dist of the moment of the pop), which
  // happens when the arming robot vertex is a cascade member that pops late with a small potential.  Written once by the
  // thread that arms, read from the next round on.
  unsigned int goal_time[6];
  unsigned int deep_labels;     // k_cvp_epilogue: finite labels whose pop time has more than 3 cascade levels (exact; informational)
  unsigned int pool_top;        // bump allocator of the level pool (words)
  unsigned int pool_overflow;   // a deep label did not fit into the level pool: reported as an error by the host
  int robot_left;               // robot-face vertices not yet settled
  unsigned int query;           // batch: query index owned by the group
  unsigned long long rounds, recomputes, settled;
  unsigned long long skipped;   // candidate-rounds that kept their label without a recompute (clean-candidate skip)
  unsigned int strict_armed;    // wavefronts that had to arm the strict back-step rule
  unsigned int watchdog;        // a wavefront hit the round watchdog (reported as non-convergence)
  unsigned long long t_work, t_flush, t_sync;   // clock cycles of thread 0 of the group: candidate loop / stage flush / barrier
  unsigned int barrier[2];      // grid_barrier state (whole-grid groups only)
  unsigned long long t_ph[8];   // phase cycles of thread 0 inside one candidate iteration (debug)
};

template <int CS>
__device__ __forceinline__ void group_sync(unsigned int* bar = nullptr) {
  if constexpr (CS == 1) {
    __syncthreads();
  } else if constexpr (CS == 0) {
    (void)bar;
    cg::this_grid().sync();   // a hand-rolled single-fence barrier measured slower (7.5k vs 5.1k cycles per round)
  } else {
    cg::this_cluster().sync();
  }
}

// per-CTA staging of appends to the next candidate list
template <int CAP_>
struct StageT {
  static constexpr int CAP = CAP_;
  static constexpr int SW_CAP = 1024;     // stage slots that take part in the in-round sweeps
  uint32_t buf[CAP];
  unsigned int n;
  unsigned int base;
  unsigned int m_tau;
  unsigned int lo;
};
using Stage = StageT<3072>;
// in-round sweeps (run_band_rounds_sub8<.., true>): per stage slot, the version of its vertex at the last evaluation
// and a copy of its label; the per-sweep dirty list.  Lives in the shared memory of the whole-grid kernel only.
struct SweepStage {
  uint32_t seen[Stage::SW_CAP];
  uint4 lab[Stage::SW_CAP];     // the slot vertex's own label (only its owner CTA writes it during a round)
  uint16_t dl[Stage::SW_CAP];
  unsigned int dn[2];           // dirty-list length, double-buffered over sweeps
};
constexpr uint32_t SEEN_NEVER = 0xffffffffu;

__device__ __forceinline__ unsigned int stage_push(Stage& st, uint32_t v, uint32_t* list_next, unsigned int* count_next) {
  const unsigned int p = atomicAdd(&st.n, 1u);
  if (p < Stage::CAP) st.buf[p] = v;
  else list_next[atomicAdd(count_next, 1u)] = v;  // overflow: straight to global
  return p;
}
// same, and registers the slot for the in-round sweeps with the version its vertex had at the last evaluation
__device__ __forceinline__ void stage_push_seen(Stage& st, SweepStage& ss, uint32_t v, uint32_t seen, const uint4& label_bits,
                                                uint32_t* list_next, unsigned int* count_next) {
  const unsigned int p = stage_push(st, v, list_next, count_next);
  if (p < Stage::SW_CAP) { ss.seen[p] = seen; ss.lab[p] = label_bits; }
}

// flush the CTA stage to the global list (all threads of the CTA call this)
template <class S>
__device__ __forceinline__ void stage_flush(S& st, uint32_t* list_next, unsigned int* count_next,
                                            unsigned int* g_m_tau, unsigned int* g_lo) {
  __syncthreads();
  const unsigned int n = st.n < (unsigned)S::CAP ? st.n : (unsigned)S::CAP;
  if (threadIdx.x == 0) {
    st.base = n ? atomicAdd(count_next, n) : 0u;
    if (st.m_tau != INF_BITS) atomicMin(g_m_tau, st.m_tau);
    if (st.lo != INF_BITS) atomicMin(g_lo, st.lo);
  }
  __syncthreads();
  const unsigned int base = st.base;
  for (unsigned int i = threadIdx.x; i < n; i += blockDim.x) list_next[base + i] = st.buf[i];
  __syncthreads();
  if (threadIdx.x == 0) { st.n = 0; st.m_tau = INF_BITS; st.lo = INF_BITS; }
  // no barrier needed here: the group barrier that follows every flush orders the reset
  // before the next round's pushes
}

// -----------------------------------------------------------------------------
// The round loop.  Preconditions (established by the caller inside the kernel,
// followed by a group_sync): states of seeds written, mark[seed] = MARK_FIXED,
// list0 holds the first candidates (mark = MARK_CAND), ctl->count[0] = |list0|,
// ctl->count[1] = ctl->count[2] = 0, ctl->m_tau[0] = ctl->lo[0] = INF,
// ctl->m_tau[1] = ctl->lo[1] = INF, ctl->m_tau[2] = 0, ctl->lo[2] = bits(seed_min).
//
// Problem P provides
//   bool  recompute(c, band_end, goal, d_old, tau_old, &d_new, &tau_new)  -> true if changed
//         (writes state/aux itself)
//   void  activate(c, push)   calls push(x) for every vertex x that shares a face/edge with c
//   bool  eligible(x)         may x ever receive a label
// -----------------------------------------------------------------------------
template <int CS, class P>
__device__ void run_band_rounds(P& prob, GroupCtl* ctl, uint32_t* list0, uint32_t* list1, uint32_t* mark,
                                Stage& st, const float delta, const uint32_t gthreads, const uint32_t gtid,
                                const int has_robot, const uint32_t r0, const uint32_t r1, const uint32_t r2,
                                const double goal_dist_offset, const volatile int* cancel_flag,
                                const float band_end_init, const uint32_t max_rounds) {
  float band_end_prev = band_end_init;  // > every seed potential: seeds are available from round 0
  unsigned long long my_recomputes = 0, my_settled = 0, my_skipped = 0;
  float lo_best = -1.0f; int stagnant = 0;       // best (largest) earliest-unsettled pop time seen so far
  prob.strict = 0;
  uint32_t r = 0;
  for (;; ++r) {
    const uint32_t slot = r % 3, prev = (r + 2) % 3, next = (r + 1) % 3;
    const unsigned int n = __ldcg(&ctl->count[slot]);
    const float m_prev = __uint_as_float(__ldcg(&ctl->m_tau[prev]));
    const float lo_prev = __uint_as_float(__ldcg(&ctl->lo[prev]));
    const unsigned int goal_b = __ldcg(&ctl->goal_ring[r & 1]);
    const float goal = __uint_as_float(goal_b);
    if constexpr (P::HAS_GOAL_TIME) if (has_robot && goal_b != INF_BITS) {
      prob.goal_t.a1 = __uint_as_float(__ldcg(&ctl->goal_time[0])); prob.goal_t.root = __ldcg(&ctl->goal_time[1]);
      prob.goal_t.a2 = __uint_as_float(__ldcg(&ctl->goal_time[2])); prob.goal_t.a3 = __uint_as_float(__ldcg(&ctl->goal_time[3]));
      prob.goal_t.ext = __ldcg(&ctl->goal_time[4]); prob.goal_t.self = __ldcg(&ctl->goal_time[5]);
    }
    const unsigned int stop = __ldcg(&ctl->stop_ring[r & 1]);
    if (n == 0 || stop || r > max_rounds) break;   // r is group-uniform: the watchdog cannot deadlock the barrier
    if (r > 0 && __float_as_uint(m_prev) == INF_BITS &&
        (__float_as_uint(lo_prev) == INF_BITS || lo_prev > goal)) break;
    // stagnation watch (all values are group-uniform): labels keep changing but the earliest unsettled pop
    // time does not move -> a dependency cycle between a trigger and its back-step child; arm the strict rule
    if (r > 0 && __float_as_uint(m_prev) != INF_BITS && !(lo_prev > lo_best)) { if (++stagnant >= P::STAGNATION) prob.strict = 1; }
    else { stagnant = 0; if (lo_prev > lo_best) lo_best = lo_prev; }
    float band_end = lo_prev + delta;
    if (!(band_end > band_end_prev)) band_end = band_end_prev;
    uint32_t* list_r = (r & 1) ? list1 : list0;
    uint32_t* list_n = (r & 1) ? list0 : list1;
    if (gtid == 0) {
      ctl->count[(r + 2) % 3] = 0;         // list r+2's counter (free during this round)
      ctl->m_tau[next] = INF_BITS;
      ctl->lo[next] = INF_BITS;
      atomicMin(&ctl->goal_ring[(r + 1) & 1], goal_b);                 // carry the cutoff into the next round
      ctl->stop_ring[(r + 1) & 1] = (stop || (cancel_flag && (r & 31) == 0 && *cancel_flag)) ? 1u : 0u;
    }
#ifdef MNB_EMU_ACTIVE   // round trace on the CPU interpreter of the kernels (tests/emu, MNB_EMU_TRACE=1): list length and progress per round
    if (gtid == 0 && getenv("MNB_EMU_TRACE")) fprintf(stderr, "[round %u] list %u m_prev %g lo_prev %g strict %d\n", r, n, m_prev, lo_prev, prob.strict);
#endif
    bool skip_ok = false;
    if constexpr (P::CAN_SKIP) skip_ok = prob.skip_clean && !has_robot && (P::SKIP_IN_STRICT || !prob.strict) && __float_as_uint(delta) == INF_BITS;
    float my_mtau = __uint_as_float(INF_BITS), my_lo = __uint_as_float(INF_BITS);
    // the evaluation of one candidate: recompute, stamps of the clean-candidate skip, re-staging, activation of the neighbours
    auto evaluate = [&](const uint32_t c, const Label& old, const bool nf) {
      const float tau = old.t.a1;
      float nd, ntau;
      my_recomputes++;
      if constexpr (P::CAN_SKIP) prob.deferred_flag = false;
      const bool changed = prob.recompute(c, band_end, goal, r, old, nd, ntau);
      if (changed) my_mtau = fminf(my_mtau, fminf(tau, ntau));
      if constexpr (P::CAN_SKIP) if (skip_ok) {
        __stcg(&prob.last_eval[c], prob.deferred_flag ? 0u : r + 1u);
        if (changed) prob.activate(c, [&](uint32_t x) { __stcg(&prob.dirty_round[x], r + 1u); });
      }
      if (!nf) my_lo = fminf(my_lo, ntau);      // smallest pop time still in flight: the band follows it
      stage_push(st, c, list_n, &ctl->count[next]);
      // a vertex that holds a finite label pulls its neighbours into the candidate set (once)
      if (__float_as_uint(nd) != INF_BITS && __ldcg(&mark[c]) == MARK_CAND) {
        mark[c] = MARK_CAND_ACT;
        prob.activate(c, [&](uint32_t x) {
          if (__ldcg(&mark[x]) == MARK_NONE && prob.eligible(x) && atomicCAS(&mark[x], MARK_NONE, MARK_CAND) == MARK_NONE)
            stage_push(st, x, list_n, &ctl->count[next]);
        });
      }
    };
    bool two_phase = false;
    if constexpr (P::CAN_SKIP) two_phase = skip_ok;
    if (two_phase) {
      if constexpr (P::CAN_SKIP) {
        // With the clean-candidate skip two thirds of the candidates of a round keep their label; one thread per list
        // entry would leave the recomputing lanes scattered over all warps (a warp is as slow as its slowest lane).  So the
        // CTA first CLASSIFIES its share of the list (settled / clean / needs an evaluation) and queues the last kind in
        // shared memory, then evaluates the queue with full warps.  Same decisions, same stamps, same results.
        constexpr unsigned int WQ_CAP = 2048;
        __shared__ uint32_t wq[WQ_CAP];
        __shared__ unsigned int wq_n;
        if (threadIdx.x == 0) wq_n = 0;
        __syncthreads();
        auto drain = [&]() {                                 // called by all threads of the CTA, right after a barrier
          const unsigned int m = wq_n;
          for (unsigned int k = threadIdx.x; k < m; k += blockDim.x) {
            const uint32_t c = wq[k];
            evaluate(c, prob.load_label(c), prob.never_fixed(c));
          }
          __syncthreads();
          if (threadIdx.x == 0) wq_n = 0;
          __syncthreads();
        };
        unsigned int chunks = 0;
        for (unsigned int b = gtid - threadIdx.x; b < n; b += gthreads) {
          const unsigned int i = b + threadIdx.x;
          if (i < n) {
            const uint32_t c = __ldcg(&list_r[i]);
            const Label old = prob.load_label(c);
            const float tau = old.t.a1;
            const bool nf = prob.never_fixed(c);
            if (tau < m_prev && tau < band_end_prev && (!nf || __float_as_uint(m_prev) == INF_BITS)) {
              mark[c] = MARK_FIXED; my_settled++;            // converged prefix (no robot bookkeeping: skip_ok excludes it)
            } else {
              const uint32_t le = __ldcg(&prob.last_eval[c]), dr = __ldcg(&prob.dirty_round[c]);
              if (le != 0u && dr < le) {                     // clean: same inputs, same label
                if (!nf) my_lo = fminf(my_lo, tau);
                my_skipped++;
                stage_push(st, c, list_n, &ctl->count[next]);
              } else {
                wq[atomicAdd(&wq_n, 1u)] = c;
              }
            }
          }
          if (++chunks == WQ_CAP / blockDim.x) { __syncthreads(); drain(); chunks = 0; }     // CTA-uniform: a chunk queues <= blockDim entries
        }
        __syncthreads();
        drain();
      }
    } else
    for (unsigned int i = gtid; i < n; i += gthreads) {
      const uint32_t c = __ldcg(&list_r[i]);
      const Label old = prob.load_label(c);
      const float d = old.d, tau = old.t.a1;
      // a vertex that is never fixed (inflation: invalid vertices pop without being fixed, inflation_layer.cpp:417-422) keeps
      // receiving updates from faces that fire AFTER its own pop: its label is not a function of earlier events only, so it
      // stays a candidate until a whole round went by without any change, and it does not hold the band back
      const bool nf = prob.never_fixed(c);
      if (tau < m_prev && tau < band_end_prev && (!nf || __float_as_uint(m_prev) == INF_BITS)) {
        // converged prefix: the sequential algorithm has popped c with exactly this label
        mark[c] = MARK_FIXED;
        my_settled++;
        if (has_robot && (c == r0 || c == r1 || c == r2)) {
          if (atomicSub(&ctl->robot_left, 1) == 1) {
            // c is not necessarily the last of the three in event order: take the latest pop time
            float bd = d; EvTime bt = old.t;
            const uint32_t rv[3] = {r0, r1, r2};
            for (int k = 0; k < 3; ++k) {
              const Label so = prob.load_label(rv[k]);
              if (prob.tless(bt, so.t)) { bt = so.t; bd = so.d; }
            }
            ctl->goal_time[0] = __float_as_uint(bt.a1); ctl->goal_time[1] = bt.root; ctl->goal_time[2] = __float_as_uint(bt.a2);
            ctl->goal_time[3] = __float_as_uint(bt.a3); ctl->goal_time[4] = bt.ext; ctl->goal_time[5] = bt.self;
            atomicMin(&ctl->goal_ring[(r + 1) & 1], __float_as_uint((float)((double)bd + goal_dist_offset)));
          }
        }
        continue;
      }
      evaluate(c, old, nf);
    }
    {
      my_mtau = fminf(my_mtau, prob.deferred_m);      // deferred back-steps are pending changes
      prob.deferred_m = __uint_as_float(INF_BITS);
      const unsigned int wm = __reduce_min_sync(0xffffffffu, __float_as_uint(my_mtau));
      const unsigned int wl = __reduce_min_sync(0xffffffffu, __float_as_uint(my_lo));
      if ((threadIdx.x & 31) == 0) {
        if (wm != INF_BITS) atomicMin(&st.m_tau, wm);
        if (wl != INF_BITS) atomicMin(&st.lo, wl);
      }
    }
    stage_flush(st, list_n, &ctl->count[next], &ctl->m_tau[slot], &ctl->lo[slot]);
    band_end_prev = band_end;
    group_sync<CS>(ctl->barrier);
  }
  // statistics
  atomicAdd(&ctl->recomputes, my_recomputes);
  atomicAdd(&ctl->settled, my_settled);
  if (my_skipped) atomicAdd(&ctl->skipped, my_skipped);
  if (gtid == 0) {
    ctl->rounds += r;
    if (prob.strict) ctl->strict_armed += 1;
    if (r > max_rounds) ctl->watchdog = 1;
    ctl->goal_bits = min(ctl->goal_ring[0], ctl->goal_ring[1]);
  }
}

// -----------------------------------------------------------------------------
// Same round loop with 8 lanes per candidate (problem provides replay_sub8 / activate via its ELL row).
// Used by the whole-grid single-plan kernel where per-round LATENCY is what matters.
// -----------------------------------------------------------------------------
template <int CS, bool SW, class P>
__device__ void run_band_rounds_sub8(P& prob, GroupCtl* ctl, uint32_t* list0, uint32_t* list1, uint32_t* mark,
                                     Stage& st, const float delta, const uint32_t gthreads, const uint32_t gtid,
                                     const int has_robot, const uint32_t r0, const uint32_t r1, const uint32_t r2,
                                     const double goal_dist_offset, const volatile int* cancel_flag,
                                     const float band_end_init, const uint32_t max_rounds, const int n_sweeps_arg,
                                     SweepStage* ss, const uint32_t n_vertices) {
  const int n_sweeps = SW ? n_sweeps_arg : 0;
  bool rescanned = false;
  float band_end_prev = band_end_init;
  unsigned long long my_recomputes = 0, my_settled = 0, my_skipped = 0;
  float lo_best = -1.0f; int stagnant = 0;       // best (largest) earliest-unsettled pop time seen so far
  prob.strict = 0;
  const uint32_t j = threadIdx.x & 7;
  const uint32_t nblk = gthreads / blockDim.x, blk = gtid / blockDim.x;   // CTAs of this group / my CTA's rank in it
  uint32_t r = 0;
  for (;; ++r) {
    const uint32_t slot = r % 3, prev = (r + 2) % 3, next = (r + 1) % 3;
    const unsigned int n = __ldcg(&ctl->count[slot]);
    const float m_prev = __uint_as_float(__ldcg(&ctl->m_tau[prev]));
    const float lo_prev = __uint_as_float(__ldcg(&ctl->lo[prev]));
    const unsigned int goal_b = __ldcg(&ctl->goal_ring[r & 1]);
    const float goal = __uint_as_float(goal_b);
    if constexpr (P::HAS_GOAL_TIME) if (has_robot && goal_b != INF_BITS) {
      prob.goal_t.a1 = __uint_as_float(__ldcg(&ctl->goal_time[0])); prob.goal_t.root = __ldcg(&ctl->goal_time[1]);
      prob.goal_t.a2 = __uint_as_float(__ldcg(&ctl->goal_time[2])); prob.goal_t.a3 = __uint_as_float(__ldcg(&ctl->goal_time[3]));
      prob.goal_t.ext = __ldcg(&ctl->goal_time[4]); prob.goal_t.self = __ldcg(&ctl->goal_time[5]);
    }
    const unsigned int stop = __ldcg(&ctl->stop_ring[r & 1]);
    // the round in which the goal cutoff first becomes visible must run even if nothing else is left to do: it puts the
    // vertices that settled beyond the cutoff back into the list (see below)
    const bool need_rescan = has_robot && goal_b != INF_BITS && !rescanned;
    if (stop || r > max_rounds) break;             // r is group-uniform: the watchdog cannot deadlock the barrier
    if (!need_rescan && n == 0) break;
    if (!need_rescan && r > 0 && __float_as_uint(m_prev) == INF_BITS &&
        (__float_as_uint(lo_prev) == INF_BITS || lo_prev > goal)) break;
    // stagnation watch (all values are group-uniform): labels keep changing but the earliest unsettled pop
    // time does not move -> a dependency cycle between a trigger and its back-step child; arm the strict rule
    if (r > 0 && __float_as_uint(m_prev) != INF_BITS && !(lo_prev > lo_best)) { if (++stagnant >= STAGNATION_ROUNDS) prob.strict = 1; }
    else { stagnant = 0; if (lo_prev > lo_best) lo_best = lo_prev; }
    // the sweeps work on the first SW_CAP stage slots of a CTA: on very long fronts (tens of millions of vertices) the
    // band is narrowed so that a CTA's share of the list still fits (group-uniform, exactness does not depend on it)
#ifdef MNB_EMU_ACTIVE   // round trace on the CPU interpreter of the kernels (tests/emu, MNB_EMU_TRACE=1)
    if (gtid == 0 && getenv("MNB_EMU_TRACE")) fprintf(stderr, "[round %u] list %u m_prev %g lo_prev %g strict %d\n", r, n, m_prev, lo_prev, prob.strict);
#endif
    float delta_r = delta;
    if constexpr (SW) {
      const float fit = (float)nblk * (0.8f * (float)Stage::SW_CAP);
      if ((float)n > fit) delta_r = fmaxf(0.25f * delta, delta * fit / (float)n);
    }
    float band_end = lo_prev + delta_r;
    if (!(band_end > band_end_prev)) band_end = band_end_prev;
    uint32_t* list_r = (r & 1) ? list1 : list0;
    uint32_t* list_n = (r & 1) ? list0 : list1;
    if (gtid == 0) {
      ctl->count[(r + 2) % 3] = 0;
      ctl->m_tau[next] = INF_BITS;
      ctl->lo[next] = INF_BITS;
      atomicMin(&ctl->goal_ring[(r + 1) & 1], goal_b);                 // carry the cutoff into the next round
      ctl->stop_ring[(r + 1) & 1] = (stop || (cancel_flag && (r & 31) == 0 && *cancel_flag)) ? 1u : 0u;
    }
    // Clean-candidate skip (group-uniform switch): a label is a pure function of the source labels, the band end (only
    // through sources beyond it), the goal cutoff and -- in strict mode -- the round number.  Plans with a goal cutoff
    // and strict rounds recompute everything; otherwise a candidate none of whose sources was re-labelled in or after the
    // round of its own last evaluation, and whose relevant sources beyond the band end are still beyond it, keeps its
    // label without being recomputed.
    bool skip_ok = false;
    if constexpr (P::CAN_SKIP) skip_ok = prob.skip_clean && !has_robot && !prob.strict;
    // Goal cutoff (cvp:754 / dijkstra:299) with a band wider than goal_dist_offset: labels computed before the cutoff
    // is known may rest on sources that turn out to lie beyond it.  Once it is known, (1) vertices beyond it never
    // settle any more -- they are recomputed under the cutoff until nothing changes -- and (2) the ones that had already
    // settled are put back into the candidate list by one sweep over the vertex array (their labels only depend on
    // vertices inside the cutoff, which are unaffected, so a single recompute repairs them).
    const float settle_cap = (has_robot && goal_b != INF_BITS) ? nextafterf(goal, __uint_as_float(INF_BITS)) : __uint_as_float(INF_BITS);
    bool requeued = false;
    if (need_rescan) {
      rescanned = true;
      for (uint32_t v = gtid; v < n_vertices; v += gthreads) {
        if (__ldcg(&mark[v]) != MARK_FIXED) continue;
        const float tv = __uint_as_float(__ldcg(&prob.state[v]).y);
        if (tv > goal) {
          mark[v] = MARK_CAND_ACT;
          if constexpr (SW) stage_push_seen(st, *ss, v, SEEN_NEVER, __ldcg(&prob.state[v]), list_n, &ctl->count[next]);
          else stage_push(st, v, list_n, &ctl->count[next]);
          requeued = true;
        }
      }
    }
#ifdef MNB_GRID_TIMING
    const long long tp0 = clock64();
#endif
    float my_mtau = requeued ? goal : __uint_as_float(INF_BITS), my_lo = requeued ? goal : __uint_as_float(INF_BITS);   // a pending change
    // One evaluation of candidate c by its 8-lane group (every lane of the WARP calls this; idle groups pass
    // has = false so that the sub-warp shuffles can use compile-time full masks).  `fresh` = main pass (c comes from
    // the round's list and is pushed to the stage); otherwise c already sits in the stage (in-round sweep).
    auto evaluate = [&](bool has, const uint32_t c, const Label& old, const int4& ix, const float4& w, const uint32_t mk,
                        const uint32_t v0, const bool fresh, const uint32_t slot) {
      const float d = old.d, tau = old.t.a1;
      float nd; EvTime nt; int deg; uint32_t mk1 = MARK_FIXED, mk2 = MARK_FIXED; float excl = 0.0f;
      prob.replay_sub8(c, j, has, ix, w, band_end, goal, r, mark, old.t, nd, nt, deg, mk1, mk2, excl);
      const bool changed = has && (__float_as_uint(nd) != __float_as_uint(d) || !prob.teq(nt, old.t));
      if constexpr (P::CAN_SKIP) if (skip_ok) {
        // stamps of the clean-candidate skip: c was evaluated in this round; its face neighbours have a source that was
        // re-labelled in this round (plain stores: every writer of a round stores the same value, rounds are barrier-ordered)
        if (has && j == 0) { __stcg(&prob.last_eval[c], r + 1u); __stcg(&prob.excl_min[c], __float_as_uint(excl)); }
        if (changed) {
          if (ix.x != -1 && deg <= 8) { __stcg(&prob.dirty_round[ix.x], r + 1u); if constexpr (P::TWO_SOURCES) __stcg(&prob.dirty_round[ix.y], r + 1u); }
          if (j == 0 && deg > 8) prob.activate(c, [&](uint32_t x) { __stcg(&prob.dirty_round[x], r + 1u); });
        }
      }
#ifdef MNB_EMU_ACTIVE
      if (has && j == 0 && getenv("MNB_DBG_V") && (c == (uint32_t)atoi(getenv("MNB_DBG_V")) || (getenv("MNB_DBG_V2") && c == (uint32_t)atoi(getenv("MNB_DBG_V2")))))
        fprintf(stderr, "[r%u %s] c=%u old d=%.9g t=(%.9g,%u,%.9g,%.9g,ext %x) -> nd=%.9g nt=(%.9g,%u,%.9g,%.9g,ext %x) changed=%d strict=%d\n", r, fresh ? "main" : "sweep", c, old.d, old.t.a1, old.t.root, old.t.a2, old.t.a3, old.t.ext, nd, nt.a1, nt.root, nt.a2, nt.a3, nt.ext, (int)changed, prob.strict);
#endif
      if (has && j == 0) {
        my_recomputes++;
        if (changed) {
          prob.store_label(c, nd, nt, __float_as_uint(d) != INF_BITS, r);
          my_mtau = fminf(my_mtau, fminf(tau, nt.a1));
        }
        my_lo = fminf(my_lo, nt.a1);
        if constexpr (SW) {
          if (fresh) stage_push_seen(st, *ss, c, v0, prob.pack_label(c, nd, nt), list_n, &ctl->count[next]);
          else if (changed) ss->lab[slot] = prob.pack_label(c, nd, nt);
        } else {
          stage_push(st, c, list_n, &ctl->count[next]);
        }
      }
      if constexpr (SW) if (n_sweeps > 0) {
        // tell the vertices that read c's label (its face neighbours) that it changed by bumping their version.
        // No fence / release-acquire pairing on purpose: the sweeps are opportunistic -- a neighbour that polls the
        // bump but still reads the old label merely misses one in-round update; the next round's main pass
        // recomputes every candidate and the change is accounted in m_tau, so exactness never depends on it.
        __syncwarp();
        if (changed) {
          if (ix.x != -1 && deg <= 8) { atomicAdd(&prob.ver[ix.x], 1u); if constexpr (P::TWO_SOURCES) atomicAdd(&prob.ver[ix.y], 1u); }
          if (j == 0 && deg > 8) prob.activate(c, [&](uint32_t x) { atomicAdd(&prob.ver[x], 1u); });
        }
      }
      if (has && __float_as_uint(nd) != INF_BITS && mk == MARK_CAND) {
        // every lane pulls the two source vertices of its own corner into the candidate set; their marks
        // were fetched together with their labels, so only genuinely new vertices cost an atomic
        if (ix.x != -1) {
          if (!prob.prefetch_marks) { mk1 = __ldcg(&mark[ix.x]); if (P::TWO_SOURCES) mk2 = __ldcg(&mark[ix.y]); }
          if (mk1 == MARK_NONE && prob.eligible((uint32_t)ix.x) && atomicCAS(&mark[ix.x], MARK_NONE, MARK_CAND) == MARK_NONE)
            { if constexpr (SW) stage_push_seen(st, *ss, (uint32_t)ix.x, SEEN_NEVER, state_inf(), list_n, &ctl->count[next]); else stage_push(st, (uint32_t)ix.x, list_n, &ctl->count[next]); }
          if (P::TWO_SOURCES && mk2 == MARK_NONE && prob.eligible((uint32_t)ix.y) && atomicCAS(&mark[ix.y], MARK_NONE, MARK_CAND) == MARK_NONE)
            { if constexpr (SW) stage_push_seen(st, *ss, (uint32_t)ix.y, SEEN_NEVER, state_inf(), list_n, &ctl->count[next]); else stage_push(st, (uint32_t)ix.y, list_n, &ctl->count[next]); }
        }
        if (j == 0 && deg > 8)
          prob.activate(c, [&](uint32_t x) {
            if (__ldcg(&mark[x]) == MARK_NONE && prob.eligible(x) && atomicCAS(&mark[x], MARK_NONE, MARK_CAND) == MARK_NONE)
              { if constexpr (SW) stage_push_seen(st, *ss, x, SEEN_NEVER, state_inf(), list_n, &ctl->count[next]); else stage_push(st, x, list_n, &ctl->count[next]); }
          });
        if (j == 0) mark[c] = MARK_CAND_ACT;
      }
    };
    // warp-uniform trip count: every lane of the warp runs every iteration (idle groups carry has = false) so
    // that the sub-warp shuffles below can use compile-time full masks (no MATCH.ANY / WARPSYNC sequences)
    // the candidates are dealt to the CTAs of the group in equal contiguous chunks and packed into the
    // lowest warps of each CTA: a round's cost is the instruction stream of its busiest SM, so an even
    // spread (instead of filling the first CTAs completely) is what shortens the round
    // ... and dealt round-robin (candidate i -> CTA i mod nblk): the list is ordered by flush time, i.e. by how busy the
    // producing CTA was, so contiguous chunks would hand all the "hot" candidates (the ones whose labels are still
    // moving) to a few CTAs while the rest idle at the barrier
    const unsigned int cnt = n > blk ? (n - blk + nblk - 1) / nblk : 0u;
    for (unsigned int qb = (threadIdx.x >> 5) * 4u; qb < cnt; qb += (blockDim.x >> 3)) {
      const unsigned int q = qb + ((threadIdx.x & 31) >> 3);
      bool has = q < cnt;
      uint32_t c = 0;
      if (has) c = __ldcg(&list_r[(size_t)q * nblk + blk]);
      // issue the independent loads of the candidate together: its label, its ELL row, its mark (and version)
      Label old = prob.load_label(has ? c : 0u);
      int4 ix = prob.load_row_idx(has ? c : 0u, j);
      float4 w = prob.load_row_w(has ? c : 0u, j);
      const uint32_t mk = __ldcg(&mark[has ? c : 0u]);
      uint32_t v0 = 0;
      if constexpr (SW) if (n_sweeps > 0) v0 = __ldcg(&prob.ver[has ? c : 0u]);
      const float d = old.d, tau = old.t.a1;
      if (has && tau < m_prev && tau < band_end_prev && tau < settle_cap) {
        if (j == 0) {
          mark[c] = MARK_FIXED;
          my_settled++;
          if (has_robot && (c == r0 || c == r1 || c == r2)) {
            if (atomicSub(&ctl->robot_left, 1) == 1) {
              float bd = d; EvTime bt = old.t;
              const uint32_t rv[3] = {r0, r1, r2};
              for (int k = 0; k < 3; ++k) {
                const Label so = prob.load_label(rv[k]);
                if (prob.tless(bt, so.t)) { bt = so.t; bd = so.d; }
              }
              ctl->goal_time[0] = __float_as_uint(bt.a1); ctl->goal_time[1] = bt.root; ctl->goal_time[2] = __float_as_uint(bt.a2);
            ctl->goal_time[3] = __float_as_uint(bt.a3); ctl->goal_time[4] = bt.ext; ctl->goal_time[5] = bt.self;
            atomicMin(&ctl->goal_ring[(r + 1) & 1], __float_as_uint((float)((double)bd + goal_dist_offset)));
            }
          }
        }
        has = false;
      }
      if constexpr (P::CAN_SKIP) if (skip_ok && has) {
        const uint32_t le = __ldcg(&prob.last_eval[c]), dr = __ldcg(&prob.dirty_round[c]);
        const float em = __uint_as_float(__ldcg(&prob.excl_min[c]));
        if (le != 0u && dr < le && !(band_end > em)) {
          // clean: survives with its label as it is (the 8 lanes of the group agree: same loads)
          if (j == 0) {
            my_lo = fminf(my_lo, tau);
            my_skipped++;
            if constexpr (SW) stage_push_seen(st, *ss, c, v0, prob.pack_label(c, old.d, old.t), list_n, &ctl->count[next]);
            else stage_push(st, c, list_n, &ctl->count[next]);
          }
          has = false;
        }
      }
      evaluate(has, c, old, ix, w, mk, v0, true, 0u);
    }
    // ---- in-round sweeps: the CTA keeps relaxing the candidates it staged (survivors + newly activated) whose
    // inputs changed since their last evaluation, so a dependency chain advances several hops per barrier ----
#ifdef MNB_GRID_TIMING
    const long long tps = clock64();
#endif
#ifdef MNB_GRID_TIMING
    if (gtid == 0) { ctl->t_ph[0] += (unsigned long long)(tps - tp0); ctl->t_ph[2] += cnt; }
#endif
    if constexpr (SW) for (int sw = 0; sw < n_sweeps; ++sw) {
#ifdef MNB_GRID_TIMING
      const long long tq0 = clock64();
#endif
      __syncthreads();                       // stage pushes / label-cache writes of the previous phase are visible
      const unsigned int ns = min(st.n, (unsigned int)Stage::SW_CAP);
      unsigned int* dcur = &ss->dn[sw & 1];
      if (threadIdx.x == 0) ss->dn[(sw + 1) & 1] = 0;
      for (unsigned int i = threadIdx.x; i < ns; i += blockDim.x) {
        const uint32_t c = st.buf[i];
        const uint32_t v0 = __ldcg(&prob.ver[c]);
        if (v0 != ss->seen[i]) { ss->seen[i] = v0; ss->dl[atomicAdd(dcur, 1u)] = (uint16_t)i; }
      }
      __syncthreads();
      const unsigned int dn = *dcur;
#ifdef MNB_GRID_TIMING
      const long long tq1 = clock64();
#endif
#ifdef MNB_GRID_TIMING
      if (gtid == 0) { ctl->t_ph[3] += dn; ctl->t_ph[4] += ns; ctl->t_ph[5] += (unsigned long long)(tq1 - tq0); }
#endif
      for (unsigned int ib = (threadIdx.x >> 5) * 4u; ib < dn; ib += (blockDim.x >> 3)) {
        const unsigned int i = ib + ((threadIdx.x & 31) >> 3);
        const bool has = i < dn;
        const uint32_t slot = has ? ss->dl[i] : 0u;
        const uint32_t c = has ? st.buf[slot] : 0u;
        // own label from the CTA's cache, ELL row through L1: the source labels are the only L2 trip of the chain
        const Label old = has ? prob.unpack_label(c, ss->lab[slot]) : prob.unpack_label(0u, state_inf());
        int4 ix = prob.load_row_idx(c, j);
        float4 w = prob.load_row_w(c, j);
        const uint32_t mk = __ldcg(&mark[c]);
        evaluate(has, c, old, ix, w, mk, 0u, false, slot);
      }
#ifdef MNB_GRID_TIMING
      if (gtid == 0) ctl->t_ph[6] += (unsigned long long)(clock64() - tq1);
#endif
    }
    {
      my_mtau = fminf(my_mtau, prob.deferred_m);      // deferred back-steps are pending changes
      prob.deferred_m = __uint_as_float(INF_BITS);
      const unsigned int wm = __reduce_min_sync(0xffffffffu, __float_as_uint(my_mtau));
      const unsigned int wl = __reduce_min_sync(0xffffffffu, __float_as_uint(my_lo));
      if ((threadIdx.x & 31) == 0) {
        if (wm != INF_BITS) atomicMin(&st.m_tau, wm);
        if (wl != INF_BITS) atomicMin(&st.lo, wl);
      }
    }
    __syncthreads();
#ifdef MNB_GRID_TIMING
    const long long tp1 = clock64();
#endif
    stage_flush(st, list_n, &ctl->count[next], &ctl->m_tau[slot], &ctl->lo[slot]);
#ifdef MNB_GRID_TIMING
    const long long tp2 = clock64();
#endif
    band_end_prev = band_end;
    group_sync<CS>(ctl->barrier);
#ifdef MNB_GRID_TIMING
    if (gtid == 0) { const long long tp3 = clock64(); ctl->t_work += (unsigned long long)(tp1 - tp0); ctl->t_flush += (unsigned long long)(tp2 - tp1); ctl->t_sync += (unsigned long long)(tp3 - tp2); }
#endif
  }
  atomicAdd(&ctl->recomputes, my_recomputes);
  atomicAdd(&ctl->settled, my_settled);
  if (my_skipped) atomicAdd(&ctl->skipped, my_skipped);
  if (gtid == 0) {
    ctl->rounds += r;
    if (prob.strict) ctl->strict_armed += 1;
    if (r > max_rounds) ctl->watchdog = 1;
    ctl->goal_bits = min(ctl->goal_ring[0], ctl->goal_ring[1]);
  }
}

}  // namespace mnb
