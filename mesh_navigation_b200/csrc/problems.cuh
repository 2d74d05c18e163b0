// Per-algorithm "pull" recompute rules plugged into the band engine.
#pragma once
#include <type_traits>
#include "band_engine.cuh"
#include "launch.cuh"

namespace mnb {

// ---------------------------------------------------------------------------
// CVP: vertex c is recomputed from its corner records (one per incident face):
//   cor_idx[k] = {v1, v2, face, -}   v1 = next(c), v2 = next(v1) in the face's cyclic order
//   cor_w[k]   = {w(v1,v2), w(v1,c), w(v2,c), -}   edge *weights* (cvp:380-390)
// Reference: the face (v1,v2,c) updates c when the later of v1,v2 is popped and c
// is the only non-fixed vertex (cvp_mesh_planner.cpp:790-866).
//
// Event (pop) time of a vertex: the stack of water levels of band_engine.cuh (EvTime / TimeAlg / LabelStore), exact for
// cascades of any depth:
//   * a vertex whose label exceeds the pop time of the face that produced it pops at its own key (d, id)  ==  the
//     oracle's canonical heap order;
//   * the CVP unfolding update is not causal (SURVEY.md H1): a face fired at water level a1 can hand out a label
//     X <= a1 ("back-step").  Such a vertex is popped inside the cascade that runs below the water line, in key order
//     among the cascade's entries: its time keeps the trigger's levels that are > (X, c) and appends (X, c).
// ---------------------------------------------------------------------------
struct CvpProblem : LabelStore {
  static constexpr bool HAS_GOAL_TIME = true;
  EvTime goal_t;                            // pop time of the vertex that armed the goal cutoff (GroupCtl::goal_time); +inf: not armed
  const uint32_t* __restrict__ cor_ptr;
  const int4* __restrict__ cor_idx;
  const float4* __restrict__ cor_w;
  const float* __restrict__ cost;
  const uint8_t* __restrict__ invalid;  // may be null
  uint32_t* pred;    // epilogue only
  float* dir;
  int32_t* cut;
  double cost_limit;
  uint32_t s0, s1, s2;       // seed vertices (pre-fixed, cvp:719-728)
  uint32_t seed_noexpand;    // bit k: seed k pops but does not expand (cvp:757,760)
  float seed_max_d = __builtin_huge_valf();   // largest seed potential: labels above it are not seeds (filter in face_time)

  static constexpr int MAXF = 12;

  uint32_t* ver;                        // input version: bumped whenever a face neighbour is re-labelled (in-round sweeps)
  mutable float deferred_m;             // smallest trigger time of a back-step deferred in this round
  int strict;                           // set by the engine once it has detected stagnation (see backstep_ok)

  // A non-causal (back-step) label X <= T.a1 may only be taken from a trigger whose label was not
  // re-labelled during the previous round.  Without this a trigger and its own back-step child can feed
  // each other forever (a dependency cycle that has no counterpart in the sequential order); the deferred
  // update is reported as a pending change at the trigger's pop time so that nothing above it settles.
  // The rule costs ~25% more rounds, so the engine only arms it (strict) after the band has made no
  // progress for a number of rounds -- the signature of such a cycle; on causal-enough inputs it never arms.
  __device__ __forceinline__ bool backstep_ok(float X, const EvTime& T, uint32_t Tv, uint32_t round) const {
    if (!strict || X > T.a1) return true;
    if (__ldcg(&chg[Tv]) < round) return true;
    deferred_m = fminf(deferred_m, T.a1);
    return false;
  }
  __device__ __forceinline__ static bool eligible(uint32_t x, const float* cost, const uint8_t* invalid, double cost_limit) {
    if (invalid && invalid[x]) return false;        // cvp:785 (no face with an invalid vertex)
    return !((double)cost[x] >= cost_limit);        // cvp:802,825,848
  }
  __device__ __forceinline__ bool eligible(uint32_t x) const { return eligible(x, cost, invalid, cost_limit); }
  __device__ __forceinline__ static bool never_fixed(uint32_t) { return false; }
  __device__ __forceinline__ int seed_index(uint32_t v) const { return v == s0 ? 0 : (v == s1 ? 1 : (v == s2 ? 2 : -1)); }

  template <class F>
  __device__ __forceinline__ void activate(uint32_t c, F push) const {
    const uint32_t kb = cor_ptr[c], ke = cor_ptr[c + 1];
    for (uint32_t k = kb; k < ke; ++k) {
      const int4 ix = __ldg(&cor_idx[k]);
      push((uint32_t)ix.x);
      push((uint32_t)ix.y);
    }
  }

  // does the vertex with label L expand when it pops?  cvp:754: not if it lies beyond goal_dist -- the goal_dist of the
  // moment it pops: a vertex that popped before the cutoff was armed expanded whatever its potential
  __device__ __forceinline__ bool expands(const Label& L, float goal) const { return !(L.d > goal && !tless(L.t, goal_t)); }
  // pop time T of the face with sources v1, v2 (= the pop of Tv); false if the face cannot fire.  PLAIN: a and b are one-level
  // times (ev_normal); the later source is then selected by value, so that its constant upper levels fold away (through a
  // reference to one of the two, they stay in memory, and so do the out-of-line comparisons they would need)
  template <bool PLAIN = false>
  __device__ __forceinline__ bool face_time(uint32_t c, uint32_t v1, uint32_t v2, const Label& a, const Label& b, float band_end,
                                            float goal, EvTime& T, uint32_t& Tv) const {
    if (!(a.d < band_end) || !(b.d < band_end)) return false;
    if (invalid && (invalid[v1] || invalid[v2])) return false;
    const bool v1_later = tless(b.t, a.t);
    if (a.d <= seed_max_d || b.d <= seed_max_d) {               // (cheap filter: only labels this small can be seeds)
      const int i1 = seed_index(v1), i2 = seed_index(v2);
      if (i1 >= 0 || i2 >= 0) {
        // Seeds are fixed BEFORE they pop (cvp:719-728).  The face fires at the pop of a source that expands while the other
        // source is already fixed: a seed always is, a normal vertex once it has popped.  With a seed and a normal vertex v
        // that is the pop of v -- even if v pops before the seed does (a neighbour closer to the goal point than the farthest
        // seed; found by the randomised tests) -- or, if v does not expand, the seed's own pop when it comes later.
        const bool e1 = expands(a, goal) && !(i1 >= 0 && ((seed_noexpand >> i1) & 1u));
        const bool e2 = expands(b, goal) && !(i2 >= 0 && ((seed_noexpand >> i2) & 1u));
        const bool fire1 = e1 && (i2 >= 0 || v1_later), fire2 = e2 && (i1 >= 0 || !v1_later);
        if (!fire1 && !fire2) return false;
        const bool use1 = fire1 && (!fire2 || !v1_later);       // both: the earlier pop
        T = use1 ? a.t : b.t; Tv = use1 ? v1 : v2;
        return !names(T, c);
      }
    }
    std::conditional_t<PLAIN, const Label, const Label&> L = v1_later ? a : b;   // two normal sources: the later pop, if that vertex expands
    if (names(L.t, c)) return false;                            // the face fires inside a cascade of c itself (LabelStore::names)
    if (!expands(L, goal)) return false;
    T = L.t; Tv = v1_later ? v1 : v2;
    return true;
  }

  __device__ __forceinline__ bool corner_time(uint32_t c, uint32_t k, float band_end, float goal, EvTime& T, uint32_t& Tv, float& u1, float& u2) const {
    const int4 ix = __ldg(&cor_idx[k]);
    const Label a = load_label((uint32_t)ix.x), b = load_label((uint32_t)ix.y);
    u1 = a.d; u2 = b.d;
    return face_time(c, (uint32_t)ix.x, (uint32_t)ix.y, a, b, band_end, goal, T, Tv);
  }

  // predecessors_/direction_/cutting_faces_ of the winning face (cvp:493-517), literal acos form; a null output is skipped.
  // ix / w: the face's corner record and weights (a CSR record or the same entry of the ELL row)
  __device__ __forceinline__ void write_aux(uint32_t c, const int4& ix, const float4& w, float wu1, float wu2) {
    CvpResult r; r.value = 0; r.direction = 0; r.pred_sel = 1;
    cvp_update_t<true>(wu1, wu2, (double)__uint_as_float(INF_BITS), w.z, w.y, w.x, r);
    if (pred) pred[c] = r.pred_sel == 1 ? (uint32_t)ix.x : (uint32_t)ix.y;
    if (dir) dir[c] = r.direction;
    if (cut) cut[c] = ix.z;
  }
  // ... no face updated c (unreached, not eligible)
  __device__ __forceinline__ void write_aux_none(uint32_t c) {
    if (pred) pred[c] = c;
    if (dir) dir[c] = 0.0f;
    if (cut) cut[c] = -1;
  }
  // ... win: CSR corner record of the winning face, -1: none
  __device__ __forceinline__ void write_aux(uint32_t c, int win, float wu1, float wu2) {
    if (win >= 0) write_aux(c, __ldg(&cor_idx[win]), __ldg(&cor_w[win]), wu1, wu2);
    else write_aux_none(c);
  }

  // generic path for vertices with more than MAXF incident faces: repeated selection of the next
  // corner in (T, corner index) order by rescanning the corner list (O(deg^2), rare)
  __device__ __noinline__ void replay_big(uint32_t c, float band_end, float goal, uint32_t round, float& nd, EvFull& nt, int& win,
                                          float& wu1, float& wu2) const {
    const uint32_t kb = cor_ptr[c], ke = cor_ptr[c + 1];
    float cur = __uint_as_float(INF_BITS);
    EvFull tc = full_normal(cur, c);
    EvTime lastT = ev_normal(0.0f, 0); uint32_t lastK = 0; bool have_last = false;
    win = -1;
    for (;;) {
      EvTime bT = lastT; float bu1 = 0, bu2 = 0; uint32_t bk = 0, bTv = 0; bool found = false;
      for (uint32_t k = kb; k < ke; ++k) {
        EvTime T; float u1, u2; uint32_t Tv;
        if (!corner_time(c, k, band_end, goal, T, Tv, u1, u2)) continue;
        if (have_last) {
          const bool after = tless(lastT, T) || (teq(lastT, T) && k > lastK);
          if (!after) continue;
        }
        if (!found || tless(T, bT) || (teq(T, bT) && k < bk)) { bT = T; bk = k; bTv = Tv; bu1 = u1; bu2 = u2; found = true; }
      }
      if (!found) break;
      if (!less_T_full(bT, tc)) break;
      const float4 w = __ldg(&cor_w[bk]);
      CvpResult r;
      if (cvp_update_t<false>(bu1, bu2, cur, w.z, w.y, w.x, r) && backstep_ok(r.value, bT, bTv, round)) { cur = r.value; accept(c, r.value, bT, tc); win = (int)bk; wu1 = bu1; wu2 = bu2; }
      lastT = bT; lastK = bk; have_last = true;
    }
    nd = cur; nt = tc;
  }

  // event-ordered replay of the faces around c (see band_engine.cuh)
  __device__ __forceinline__ void replay(uint32_t c, float band_end, float goal, uint32_t round, float& nd, EvFull& nt, int& win,
                                         float& wu1, float& wu2) const {
    const uint32_t kb = cor_ptr[c], ke = cor_ptr[c + 1];
    win = -1; wu1 = 0.0f; wu2 = 0.0f;
    if (ke - kb > (uint32_t)MAXF) {
      replay_big(c, band_end, goal, round, nd, nt, win, wu1, wu2);
      return;
    }
    EvTime Tt[MAXF]; float U1[MAXF], U2[MAXF]; uint32_t K[MAXF], TV[MAXF];
    int n = 0;
    for (uint32_t k = kb; k < ke; ++k) {
      EvTime T; float u1, u2; uint32_t Tv;
      if (!corner_time(c, k, band_end, goal, T, Tv, u1, u2)) continue;
      Tt[n] = T; U1[n] = u1; U2[n] = u2; K[n] = k; TV[n] = Tv; ++n;
    }
    float cur = __uint_as_float(INF_BITS);
    EvFull tc = full_normal(cur, c);
    for (int i = 0; i < n; ++i) {
      int b = i;
      for (int j = i + 1; j < n; ++j)
        if (tless(Tt[j], Tt[b]) || (teq(Tt[j], Tt[b]) && K[j] < K[b])) b = j;
      const EvTime T = Tt[b]; const float u1 = U1[b], u2 = U2[b]; const uint32_t k = K[b], Tv = TV[b];
      Tt[b] = Tt[i]; U1[b] = U1[i]; U2[b] = U2[i]; K[b] = K[i]; TV[b] = TV[i];
      if (!less_T_full(T, tc)) break;   // c has been popped before this face fires
      const float4 w = __ldg(&cor_w[k]);
      CvpResult r;
      if (cvp_update_t<false>(u1, u2, cur, w.z, w.y, w.x, r) && backstep_ok(r.value, T, Tv, round)) { cur = r.value; accept(c, r.value, T, tc); win = (int)k; wu1 = u1; wu2 = u2; }
    }
    nd = cur; nt = tc;
  }

  // replay() on the ELL row ix of c (slot j = corner cor_ptr[c] + j, ell_w laid out as cor_w), for the epilogue: the same
  // face times, the same (T, corner) event order and the same accept loop, with every array index a compile-time constant
  // so that the row, its source labels and the ranks stay in registers.  The event order comes from ranks (pairwise
  // comparisons) instead of a sort.  Covered: at most 8 faces, and every source label word a plain one-level time (z = w
  // = 0: no side arrays, no level pool), so that no comparison and no accept needs an out-of-line tail -- a plain trigger
  // only ever hands out times of at most two levels.  Returns false for anything else (the caller runs replay()).
  // win: winning slot (-1: none), with its weights ww and source potentials.
  __device__ __forceinline__ bool replay_row(uint32_t c, const int4 (&ix)[ELL_W], const float4* __restrict__ ell_w, float band_end,
                                             float goal, uint32_t round, int& win, float4& ww, float& wu1, float& wu2) const {
    const float INF = __uint_as_float(INF_BITS);
    if (ix[0].w > (int)ELL_W) return false;
    // every load of the row first: its 16 source labels, and the line of its weights into L1 (read in the accept loop)
    const float4* wrow = ell_w + (size_t)c * ELL_W;
    mnb_prefetch_l1(wrow);
    uint4 sa[ELL_W], sb[ELL_W];
#pragma unroll
    for (int j = 0; j < (int)ELL_W; ++j) {
      sa[j] = state_inf(); sb[j] = state_inf();
      if (ix[j].x != ELL_EMPTY) { sa[j] = __ldcg(&state[ix[j].x]); sb[j] = __ldcg(&state[ix[j].y]); }
    }
    uint32_t flags = 0u;
#pragma unroll
    for (int j = 0; j < (int)ELL_W; ++j) flags |= sa[j].z | sa[j].w | sb[j].z | sb[j].w;
    if (flags) return false;                                       // a cascade member among the sources
    // face times: (a1, Tv) of a plain pop time; a slot that does not fire sorts last
    float A1[ELL_W], U1[ELL_W], U2[ELL_W]; uint32_t TV[ELL_W];
    int n = 0;
#pragma unroll
    for (int j = 0; j < (int)ELL_W; ++j) {
      A1[j] = INF; TV[j] = 0xffffffffu; U1[j] = 0.0f; U2[j] = 0.0f;
      if (ix[j].x == ELL_EMPTY) continue;
      const uint32_t v1 = (uint32_t)ix[j].x, v2 = (uint32_t)ix[j].y;
      Label a, b;                                                  // = unpack_label() of a word with z = w = 0
      a.d = __uint_as_float(sa[j].x); a.t = ev_normal(__uint_as_float(sa[j].y), v1);
      b.d = __uint_as_float(sb[j].x); b.t = ev_normal(__uint_as_float(sb[j].y), v2);
      EvTime T; uint32_t Tv;
      if (!face_time<true>(c, v1, v2, a, b, band_end, goal, T, Tv)) continue;
      A1[j] = T.a1; TV[j] = Tv; U1[j] = a.d; U2[j] = b.d; ++n;
    }
    // rank of slot j in (T, corner) order: for plain times tless is (a1, Tv), and equal times keep the corner order
    int rank[ELL_W];
#pragma unroll
    for (int j = 0; j < (int)ELL_W; ++j) rank[j] = 0;
#pragma unroll
    for (int i = 0; i < (int)ELL_W; ++i)
#pragma unroll
      for (int j = i + 1; j < (int)ELL_W; ++j) {
        const bool j_first = A1[j] < A1[i] || (A1[j] == A1[i] && TV[j] < TV[i]);
        rank[i] += j_first ? 1 : 0;
        rank[j] += j_first ? 0 : 1;
      }
    // the accept loop of replay()
    float cur = INF;
    EvFull tc = full_normal(cur, c);
    win = -1;
#pragma unroll
    for (int r = 0; r < (int)ELL_W; ++r) {
      if (r >= n) break;
      float a1 = 0.0f, u1 = 0.0f, u2 = 0.0f; uint32_t Tv = 0u; int k = 0;
#pragma unroll
      for (int j = 0; j < (int)ELL_W; ++j)
        if (rank[j] == r) { a1 = A1[j]; Tv = TV[j]; u1 = U1[j]; u2 = U2[j]; k = j; }
      const EvTime T = ev_normal(a1, Tv);
      if (!less_T_full(T, tc)) break;   // c has been popped before this face fires
      const float4 wr = __ldg(&wrow[k]);
      CvpResult res;
      if (cvp_update_t<false>(u1, u2, cur, wr.z, wr.y, wr.x, res) && backstep_ok(res.value, T, Tv, round)) {
        cur = res.value; accept(c, res.value, T, tc); win = k; ww = wr; wu1 = u1; wu2 = u2;
      }
    }
    return true;
  }

  // the epilogue of c through replay() on the CSR records, out of line with its own frame (replay_row's other cases)
  __device__ __noinline__ void epilogue_csr(uint32_t c, float goal) {
    int win; float nd, wu1 = 0.0f, wu2 = 0.0f; EvFull nt;
    replay(c, __uint_as_float(INF_BITS), goal, 0xfffffff0u /* final labels: nothing is deferred */, nd, nt, win, wu1, wu2);
    write_aux(c, win, wu1, wu2);
  }

  // engine hook: returns true if the label changed (and stores it)
  __device__ __forceinline__ bool recompute(uint32_t c, float band_end, float goal, uint32_t round, const Label& old, float& nd, float& ntau) {
    int win; float wu1, wu2; EvFull nf;
    replay(c, band_end, goal, round, nd, nf, win, wu1, wu2);
    const EvTime nt = finish(nf, old.t);
    ntau = nt.a1;
    if (__float_as_uint(nd) == __float_as_uint(old.d) && teq(nt, old.t)) return false;
    store_label(c, nd, nt, __float_as_uint(old.d) != INF_BITS, round);
    return true;
  }
};

// The seed face of a CVP wave as the problem reads it: its vertices s0-s2, the seeds that pop but do not expand (bit k: seed
// k, cvp:757,760) and the largest seed potential
struct SeedFace { uint32_t s[3]; uint32_t noexpand; float seed_max; };
// ... and what the seeding writes: the seed potentials, the distances of the vertices to the seed point (cvp:719-728)
struct CvpSeeds : SeedFace { float d[3]; float seed_min; };
// the seed face sf with seed point sp
__device__ __forceinline__ CvpSeeds cvp_seeds(const uint32_t* faces, const float* pos, const float* cost, const uint8_t* invalid,
                                              double cost_limit, uint32_t sf, const float* sp) {
  CvpSeeds sd;
  sd.noexpand = 0;
  for (int k = 0; k < 3; ++k) {
    const uint32_t v = faces[3 * (size_t)sf + k];
    const float dx = sp[0] - pos[3 * (size_t)v];
    const float dy = sp[1] - pos[3 * (size_t)v + 1];
    const float dz = sp[2] - pos[3 * (size_t)v + 2];
    sd.s[k] = v;
    sd.d[k] = sqrtf(dx * dx + dy * dy + dz * dz);
    if (((double)cost[v] >= cost_limit) || (invalid && invalid[v])) sd.noexpand |= (1u << k);
  }
  sd.seed_min = fminf(sd.d[0], fminf(sd.d[1], sd.d[2]));
  sd.seed_max = fmaxf(sd.d[0], fmaxf(sd.d[1], sd.d[2]));
  return sd;
}

// ---------------------------------------------------------------------------
// CVP, 8 lanes per candidate ("sub-warp pull").  Corner records live in an ELL
// table: row c = 8 slots x {v1, v2, face, deg} (one 128-byte line) and a matching
// row of weights, so the 8 lanes of a group fetch a vertex's whole 1-ring with two
// coalesced 128-byte loads.  Each lane evaluates its own face (the double-precision
// unfolding) concurrently; the reference's event order is then replayed across the
// lanes with shuffles.  Vertices with more than 8 faces take the CSR path on lane 0.
// ---------------------------------------------------------------------------

struct CvpEllProblem : CvpProblem {
  static constexpr bool TWO_SOURCES = true;   // an ELL slot names the two source vertices of a face
  // whole-grid main pass: plain causal candidates one per thread (eval_plain), the rest on 8 lanes (run_band_rounds_sub8)
  static constexpr bool PLAIN_FAST = true;
  // activation marks of the two source vertices: fetched together with their labels (whole-grid single plan: one L2 trip
  // less on the evaluation that activates, which is on the wave's critical path) or only by that one evaluation
  // (throughput-bound batches: two scattered 4-byte loads = 64 L1 wavefronts per warp less on every other evaluation)
  bool prefetch_marks;
  const int4* __restrict__ ell_idx;
  const float4* __restrict__ ell_w;
  const double4* __restrict__ ell_geo;   // {p, hc, t0a, -} per slot, precomputed from ell_w (k_corner_geo)

  // face evaluation without a current label: U = unfolded distance, X = value the reference would
  // store (U when the angle test passes, else the edge fallback).  accept(cur) <=> U < cur && X < cur.
  __device__ __forceinline__ static void eval_face(double u1, double u2, double a, double b, double c, double& U, double& X) {
    const double c_sq = c * c, b_sq = b * b, a_sq = a * a;
    const double u1_sq = u1 * u1, u2_sq = u2 * u2;
    const double sx = (c_sq + u1_sq - u2_sq) / (2 * c);
    const double sy = -sqrt(fmax(u1_sq - sx * sx, 0.0));
    const double p = (b_sq + c_sq - a_sq) / (2 * c);
    const double hc = sqrt(fmax(b_sq - p * p, 0.0));
    const double dy = hc - sy;
    const double dx = p - sx;
    const double u3tmp_sq = dx * dx + dy * dy;
    const double u3tmp = sqrt(u3tmp_sq);
    U = u3tmp;
    const double t0a = (a_sq + b_sq - c_sq) / (2 * a * b);
    const double t1a = (u3tmp_sq + b_sq - u1_sq) / (2 * u3tmp * b);
    const double t2a = (a_sq + u3tmp_sq - u2_sq) / (2 * a * u3tmp);
    int fb;
    if (fabs(t1a) > 1) fb = 1;
    else if (fabs(t2a) > 1) fb = 2;
    else if (fabs(t0a) <= 1 && acos_less(t1a, t0a) && acos_less(t2a, t0a)) { X = u3tmp; return; }   // |t0a| > 1: acos(t0a) is NaN in the reference
    else fb = acos_less(t1a, t2a) ? 1 : 2;
    X = (fb == 1) ? (u1 + b) : (u2 + a);
  }

  // The throughput form of replay_sub8's fast path: ONE thread walks the ELL row of c.  Every source label plain, no source
  // that may be a seed, and the causal collapse applies: m = min over the causal faces, c pops at (m, c).  Returns false
  // (c needs the general evaluation) for more than 8 faces, a cascade member among the sources, a possible seed, or a
  // non-causal face that may fire before c pops.  excl: smallest finite source label beyond the band end.
  // Strict rounds and an armed goal cutoff are the caller's to exclude.
  __device__ __forceinline__ static bool eval_plain(const int4* __restrict__ ell_idx, const float4* __restrict__ ell_w,
                                                    const double4* __restrict__ ell_geo, const uint8_t* __restrict__ invalid,
                                                    const uint4* state, float seed_max, float band_end, uint32_t c,
                                                    float& m, float& excl) {
    (void)ell_geo;
    const float INF = __uint_as_float(INF_BITS);
    float tmin_nc = INF;
    m = INF; excl = INF;
    for (int k = 0; k < (int)ELL_W; ++k) {
      const int4 ix = __ldg(&ell_idx[(size_t)c * ELL_W + k]);
      if (k == 0 && ix.w > (int)ELL_W) return false;
      if (ix.x == ELL_EMPTY) continue;
      const uint32_t v1 = (uint32_t)ix.x, v2 = (uint32_t)ix.y;
      const uint4 sa = __ldcg(&state[v1]), sb = __ldcg(&state[v2]);
      const float da = __uint_as_float(sa.x), db = __uint_as_float(sb.x);
      if (((sa.z | sa.w | sb.z | sb.w) >> 31) || da <= seed_max || db <= seed_max) return false;
      if (invalid && (invalid[v1] || invalid[v2])) continue;
      if (sa.x != INF_BITS && !(da < band_end)) excl = fminf(excl, da);
      if (sb.x != INF_BITS && !(db < band_end)) excl = fminf(excl, db);
      if (!(da < band_end) || !(db < band_end)) continue;
      const float ta = __uint_as_float(sa.y), tb = __uint_as_float(sb.y);
      const bool v1_later = tb < ta || (tb == ta && v2 < v1);
      const float T1 = v1_later ? ta : tb;
      const float4 w = __ldg(&ell_w[(size_t)c * ELL_W + k]);
      // the static part of the unfolding (apex of the triangle, cosine at v3) is recomputed from the three weights instead of
      // being read from the precomputed table: 256 of the 512 bytes a vertex' ELL rows occupy, and the rows -- not the
      // labels -- are what makes the hot set of a few hundred concurrent wavefronts overflow the L2 (MNB_BATCH_GEO_TABLE=1
      // at compile time restores the table read)
      double U, X;
#ifdef MNB_BATCH_GEO_TABLE
      const double2* gp = reinterpret_cast<const double2*>(ell_geo) + 2 * ((size_t)c * ELL_W + k);
      const double2 g01 = __ldg(gp), g23 = __ldg(gp + 1);
      FaceGeo fg; fg.p = g01.x; fg.hc = g01.y; fg.t0a = g23.x;
      eval_face_geo((double)da, (double)db, (double)w.z, (double)w.y, (double)w.x, fg, U, X);
#else
      eval_face((double)da, (double)db, (double)w.z, (double)w.y, (double)w.x, U, X);
#endif
      const float Xf = (float)X;
      if (Xf > T1 && U <= X) m = fminf(m, Xf); else tmin_nc = fminf(tmin_nc, T1);
    }
    return __float_as_uint(tmin_nc) == INF_BITS || tmin_nc > m;     // no non-causal face may fire first
  }

  template <class F>
  __device__ __forceinline__ void activate_lane(uint32_t c, uint32_t j, const int4& ix, int deg, F push) const {
    if (ix.x != ELL_EMPTY) { push((uint32_t)ix.x); push((uint32_t)ix.y); }
    if (j == 0 && deg > (int)ELL_W) activate(c, push);   // faces beyond the 8 ELL slots
  }

  // scalar replay on one lane (more than 8 faces, or a cascade deeper than 3 levels): returns the time to STORE (a deep
  // label that did not change keeps its pool record, LabelStore::finish)
  __device__ __noinline__ void replay_serial(uint32_t c, float band_end, float goal, uint32_t round, const EvTime& old_t, float& nd, EvTime& nt) const {
    int win; float a1, a2; EvFull nf;
    replay(c, band_end, goal, round, nd, nf, win, a1, a2);
    nt = finish(nf, old_t);
  }

  __device__ __forceinline__ int4 load_row_idx(uint32_t c, uint32_t j) const { return __ldg(&ell_idx[(size_t)c * ELL_W + j]); }
  __device__ __forceinline__ float4 load_row_w(uint32_t c, uint32_t j) const { return __ldg(&ell_w[(size_t)c * ELL_W + j]); }

  // static part of the unfolding (depends on the face's weights only): apex of the triangle and the cosine at v3.
  // Evaluated while the source labels are still in flight.
  struct FaceGeo { double p, hc, t0a; };
  __device__ __forceinline__ static FaceGeo face_geo(double a, double b, double c) {
    const double c_sq = c * c, b_sq = b * b, a_sq = a * a;
    FaceGeo g;
    g.p = (b_sq + c_sq - a_sq) / (2 * c);
    g.hc = sqrt(fmax(b_sq - g.p * g.p, 0.0));
    g.t0a = (a_sq + b_sq - c_sq) / (2 * a * b);
    return g;
  }
  // dynamic part: same arithmetic, same order of operations as eval_face / the reference
  __device__ __forceinline__ static void eval_face_geo(double u1, double u2, double a, double b, double c, const FaceGeo& g,
                                                       double& U, double& X) {
    const double c_sq = c * c, b_sq = b * b, a_sq = a * a;
    const double u1_sq = u1 * u1, u2_sq = u2 * u2;
    const double sx = (c_sq + u1_sq - u2_sq) / (2 * c);
    const double sy = -sqrt(fmax(u1_sq - sx * sx, 0.0));
    const double dy = g.hc - sy;
    const double dx = g.p - sx;
    const double u3tmp_sq = dx * dx + dy * dy;
    const double u3tmp = sqrt(u3tmp_sq);
    U = u3tmp;
    const double t1a = (u3tmp_sq + b_sq - u1_sq) / (2 * u3tmp * b);
    const double t2a = (a_sq + u3tmp_sq - u2_sq) / (2 * a * u3tmp);
    int fb;
    if (fabs(t1a) > 1) fb = 1;
    else if (fabs(t2a) > 1) fb = 2;
    else if (fabs(g.t0a) <= 1 && acos_less(t1a, g.t0a) && acos_less(t2a, g.t0a)) { X = u3tmp; return; }   // |t0a| > 1: acos(t0a) is NaN in the reference
    else fb = acos_less(t1a, t2a) ? 1 : 2;
    X = (fb == 1) ? (u1 + b) : (u2 + a);
  }

  // Every lane of the WARP calls this (groups without work pass has = false): all shuffles use the
  // compile-time full mask with width 8.  Lanes of a group return the same label.  mk1/mk2 return the
  // activation marks of the lane's two source vertices (fetched together with their labels).
  __device__ __forceinline__ void replay_sub8(uint32_t c, uint32_t j, bool has, const int4& ix, const float4& w, float band_end,
                                              float goal, uint32_t round, const uint32_t* mark, const EvTime& old_t, float& nd, EvTime& nt, int& deg_out,
                                              uint32_t& mk1, uint32_t& mk2) const {
    constexpr unsigned FULL = 0xffffffffu;
    const float INF = __uint_as_float(INF_BITS);
    const int deg = __shfl_sync(FULL, ix.w, 0, 8);
    deg_out = deg;
    bool big = has && deg > (int)ELL_W;     // (also set below when the replay meets a cascade deeper than 3 levels)
    bool valid = has && !big && ix.x != ELL_EMPTY;
    EvTime T = ev_normal(INF, 0x7fffffffu);
    uint32_t Tv = 0x7fffffffu;
    double U = 0.0, X = 0.0;
    const unsigned sh = (threadIdx.x & 31) & ~7;
    if (valid) {
      const uint32_t v1 = (uint32_t)ix.x, v2 = (uint32_t)ix.y;
      // issue the four loads, then do the label-independent half of the unfolding while they are in flight
      const uint4 sa = __ldcg(&state[v1]), sb = __ldcg(&state[v2]);
      if (prefetch_marks) { mk1 = __ldcg(&mark[v1]); mk2 = __ldcg(&mark[v2]); }
      const double2* gp = reinterpret_cast<const double2*>(ell_geo) + 2 * ((size_t)c * ELL_W + j);
      const double2 g01 = __ldg(gp), g23 = __ldg(gp + 1);
      FaceGeo g; g.p = g01.x; g.hc = g01.y; g.t0a = g23.x;
      const Label a = unpack_label(v1, sa), b = unpack_label(v2, sb);
      valid = face_time(c, v1, v2, a, b, band_end, goal, T, Tv);
      if (valid) {
        eval_face_geo((double)a.d, (double)b.d, (double)w.z, (double)w.y, (double)w.x, g, U, X);
        // back-step from a trigger that was re-labelled last round: defer (see backstep_ok)
        if (!backstep_ok((float)X, T, Tv, round)) X = (double)INF;
      }
    }
    float cur = INF;
    EvTime tc = ev_normal(INF, c);
    // Fast path (the norm on geometric weights).  A face is CAUSAL if its value exceeds its own pop time (the label it hands
    // out pops at its own key, accept_time) and U <= X (the accept test is then X < cur).  Let m = min (float)X over the
    // causal faces of c.  If every other firing face has a pop time above m, the event-ordered replay collapses to m:
    //   * the causal face i* with value m fires before c pops (T.a1 < m <= every earlier cur) and nothing lowers m later;
    //   * a non-causal face j with T_j.a1 > m comes after i* in event order (T_i*.a1 < m < T_j.a1), when c -- key <= m --
    //     has already popped: it is never applied;
    //   * rejected / unreached causal faces have float values >= m (rounding is monotone).
    // So d = m and c pops at (m, c): no ranking, no replay loop.  Faces "looking backwards" (sources farther from the seed
    // than c, T > X) are the common non-causal case and are all of the harmless kind.
    const float Xf = (float)X;
    const bool causal = valid && Xf > T.a1 && U <= X;
    float m = causal ? Xf : INF;
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) m = fminf(m, __shfl_xor_sync(FULL, m, o, 8));
    if (__all_sync(FULL, !valid || causal || T.a1 > m)) {
      cur = m; tc = ev_normal(m, c);
    } else {
      // Common case: every firing face of the warp has a plain pop time (one level, root = Tv): the event order is
      // (a1, Tv).  Cascade members (rare) take the general path on the full stacks.  Invalid lanes carry the maximal key so
      // that no validity flag has to travel with the shuffles.
      const bool plain = !valid || (T.a2 == 0.0f && T.root == Tv);
      const bool all_plain = __all_sync(FULL, plain);
      const uint32_t k1 = valid ? __float_as_uint(T.a1) : 0xffffffffu;          // pop times are >= 0: bit order = value order
      const unsigned long long hi = valid ? (((unsigned long long)k1 << 32) | T.root) : ~0ull;          // plain: root == Tv
      const unsigned long long mid = ((unsigned long long)__float_as_uint(T.a2) << 32) | __float_as_uint(T.a3);
      const unsigned long long lo = ((unsigned long long)T.ext << 32) | Tv;     // (the trigger vertex = the time's own id)
      int rank = 0;
      if (all_plain) {
        // 32-bit pass on a1 alone; two firing faces with bit-identical a1 (exact float tie between different source
        // vertices) are rare -- only then is the (a1, Tv) pass needed
        bool tie = false;
  #pragma unroll
        for (int d = 1; d < 8; ++d) {
          const int src = (int)((j + d) & 7);
          const uint32_t ok1 = __shfl_sync(FULL, k1, src, 8);
          rank += (ok1 < k1) ? 1 : 0;
          tie |= (ok1 == k1) && valid;
        }
        if (__any_sync(FULL, tie)) {
          rank = 0;
  #pragma unroll
          for (int d = 1; d < 8; ++d) {
            const int src = (int)((j + d) & 7);
            const unsigned long long ohi = __shfl_sync(FULL, hi, src, 8);
            if (ohi < hi || (ohi == hi && (uint32_t)src < j)) ++rank;
          }
        }
      } else {
  #pragma unroll
        for (int d = 1; d < 8; ++d) {
          const int src = (int)((j + d) & 7);
          const unsigned long long ohi = __shfl_sync(FULL, hi, src, 8);
          const unsigned long long omid = __shfl_sync(FULL, mid, src, 8);
          const unsigned long long olo = __shfl_sync(FULL, lo, src, 8);
          if (ohi < hi) ++rank;
          else if (ohi == hi && valid) {                  // same first level: compare the rest of the two stacks
            EvTime O; O.a1 = T.a1; O.root = T.root; O.a2 = __uint_as_float((uint32_t)(omid >> 32)); O.a3 = __uint_as_float((uint32_t)omid);
            O.ext = (uint32_t)(olo >> 32); O.self = (uint32_t)olo;
            if (tless(O, T) || (!tless(T, O) && (uint32_t)src < j)) ++rank;
          }
        }
      }
      if (!valid) rank = 99;
      const int nvalid = __popc((__ballot_sync(FULL, valid) >> sh) & 0xFFu);
      bool open = nvalid > 0;                             // c has not been popped yet and faces remain
      for (int r = 0; r < (int)ELL_W; ++r) {
        if (!__any_sync(FULL, open)) break;               // every group of the warp is done
        const unsigned who = (__ballot_sync(FULL, rank == r) >> sh) & 0xFFu;
        const int src = who ? (__ffs(who) - 1) : 0;
        const unsigned long long whi = __shfl_sync(FULL, hi, src, 8);
        unsigned long long wmid = 0, wlo = 0;
        if (!all_plain) { wmid = __shfl_sync(FULL, mid, src, 8); wlo = __shfl_sync(FULL, lo, src, 8); }
        const double Uw = __shfl_sync(FULL, U, src, 8);
        const double Xw = __shfl_sync(FULL, X, src, 8);
        if (!who) open = false;                           // ranks are dense: no face with rank r -> none beyond
        if (!open) continue;
        EvTime Tw;
        Tw.a1 = __uint_as_float((uint32_t)(whi >> 32)); Tw.root = (uint32_t)whi;
        if (all_plain) { Tw.a2 = 0.0f; Tw.a3 = 0.0f; Tw.ext = 0u; Tw.self = (uint32_t)whi; }
        else { Tw.a2 = __uint_as_float((uint32_t)(wmid >> 32)); Tw.a3 = __uint_as_float((uint32_t)wmid); Tw.ext = (uint32_t)(wlo >> 32); Tw.self = (uint32_t)wlo; }
        if (!tless(Tw, tc)) { open = false; continue; }
        const double cd = (double)cur;
        if (Uw < cd && Xw < cd) {
          cur = (float)Xw;
          if (!accept_lean(c, cur, Tw, tc)) { big = true; open = false; }   // a fourth cascade level: scalar replay below
        }
      }
    }
    if (big) {   // rare: more than 8 faces / a deep cascade -> scalar path on the group's first lane, result broadcast below
      if (j == 0) {
        // (by-reference arguments of a __noinline__ callee live in local memory: keep the address-taken copies inside this
        // rare branch, or every update of cur / tc in the hot path above becomes a local store -- 4.5x the local stores of
        // the whole kernel when that was overlooked)
        const EvTime ot = old_t; float cs; EvTime ts;
        replay_serial(c, band_end, goal, round, ot, cs, ts);
        cur = cs; tc = ts;
      }
    }
    const unsigned anybig = __ballot_sync(FULL, big);
    if (anybig) {
      cur = __shfl_sync(FULL, cur, 0, 8);
      tc.a1 = __shfl_sync(FULL, tc.a1, 0, 8); tc.a2 = __shfl_sync(FULL, tc.a2, 0, 8);
      tc.a3 = __shfl_sync(FULL, tc.a3, 0, 8); tc.ext = __shfl_sync(FULL, tc.ext, 0, 8); tc.root = __shfl_sync(FULL, tc.root, 0, 8);
    }
    nd = cur; nt = tc;
  }
};

// ---------------------------------------------------------------------------
// Inflation: multi-source FMM from the lethal set (InflationLayer::waveCostInflation,
// inflation_layer.cpp:341-491) with the Kimmel-Sethian update in float (:181-313).
//   * lethal vertices: d = 0, pre-fixed, popped first in id order (:397-402);
//   * the face (v1,v2,c) updates c when the later of v1,v2 pops (:443-470);  u3 == 0 never updates (:252);
//   * an accepted update always lowers distances_[c] (:299) but only (re)inserts c into the heap if both
//     sources are within the inflation radius (:310,:452): the label d and the heap key (= pop time) are
//     therefore tracked separately; a vertex that was never inserted never pops and is never a source;
//   * invalid vertices pop but are not fixed and do not expand (:417-422) unless lethal (fixed at :400).
// Corner weights are edge_distances (:383), record {|v1v2|, |v1c|, |v2c|}.
// ---------------------------------------------------------------------------
struct InflationProblem : LabelStore {
  static constexpr bool HAS_GOAL_TIME = false;
  static constexpr bool CAN_SKIP = true;    // clean-candidate skip in run_band_rounds (delta = inf, no goal cutoff)
  // The Sethian fallback produces trigger / back-step-child cycles on ordinary inputs (config 3: one pair oscillates for 27
  // of 41 rounds until the strict rule arms).  Arming the rule earlier (2-4 stagnant rounds) halves the round count but is
  // NOT neutral: on meshes with exact key ties (unjittered grids) the early strict rounds converge to a different label
  // (fuzz seed 51 case 56, 1 vertex) -- so the engine's threshold (STAGNATION_ROUNDS) stays, and the stagnant rounds are
  // made cheap by the clean-candidate skip instead (only the oscillating pair is recomputed).
  uint32_t* last_eval; uint32_t* dirty_round; int skip_clean;
  // In strict rounds a label also depends on the round number, but only through a deferral: an evaluation that deferred
  // nothing rests on triggers that were stable, and a trigger that is re-labelled later marks its face neighbours dirty.
  // So the skip stays valid in strict rounds as long as an evaluation that deferred is never remembered as "evaluated".
  static constexpr bool SKIP_IN_STRICT = false;   // (kept off: strict rounds are rare and recompute everything, as they always did)
  mutable bool deferred_flag;
  const uint32_t* __restrict__ cor_ptr;
  const int4* __restrict__ cor_idx;
  const float4* __restrict__ cor_wd;
  const uint4* __restrict__ cor_eid;    // {edge(v1,v2), edge(v1,c), edge(v2,c), -} per corner record
  const uint8_t* __restrict__ invalid;  // may be null
  mutable float deferred_m;
  int strict;
  float max_distance;

  static constexpr int MAXF = 12;

  __device__ __forceinline__ bool backstep_ok(float X, const EvTime& T, uint32_t Tv, uint32_t round) const {   // see CvpProblem
    if (!strict || X > T.a1) return true;
    if (__ldcg(&chg[Tv]) < round) return true;
    deferred_m = fminf(deferred_m, T.a1);
    deferred_flag = true;                 // this evaluation depends on the round number: it must be repeated (clean skip)
    return false;
  }
  __device__ __forceinline__ bool eligible(uint32_t) const { return true; }   // no cost / validity test on the target
  __device__ __forceinline__ bool never_fixed(uint32_t c) const { return invalid && invalid[c]; }   // pops, but is not fixed (:417-422)

  template <class F>
  __device__ __forceinline__ void activate(uint32_t c, F push) const {
    const uint32_t kb = cor_ptr[c], ke = cor_ptr[c + 1];
    for (uint32_t k = kb; k < ke; ++k) {
      const int4 ix = __ldg(&cor_idx[k]);
      push((uint32_t)ix.x);
      push((uint32_t)ix.y);
    }
  }

  __device__ __forceinline__ bool corner_time(uint32_t c, uint32_t k, float band_end, EvTime& T, uint32_t& Tv, float& u1, float& u2) const {
    const int4 ix = __ldg(&cor_idx[k]);
    const uint32_t v1 = (uint32_t)ix.x, v2 = (uint32_t)ix.y;
    const Label a = load_label(v1), b = load_label(v2);
    u1 = a.d; u2 = b.d;
    // a source must get fixed: it is lethal (d == 0) or it is (re)inserted at some point (finite pop time)
    if (__float_as_uint(a.t.a1) == INF_BITS || __float_as_uint(b.t.a1) == INF_BITS) return false;
    if (!(a.t.a1 < band_end) || !(b.t.a1 < band_end)) return false;
    const bool l1 = (u1 == 0.0f), l2 = (u2 == 0.0f);
    const bool i1 = invalid && invalid[v1], i2 = invalid && invalid[v2];
    if ((i1 && !l1) || (i2 && !l2)) return false;           // popped but never fixed (:417)
    const bool v1_later = tless(b.t, a.t);
    if (l1 && l2) {                                          // both pre-fixed: first one that expands
      const bool e1 = !i1, e2 = !i2;
      if (!e1 && !e2) return false;
      const bool use1 = e1 && (!e2 || !v1_later);
      T = use1 ? a.t : b.t; Tv = use1 ? v1 : v2;
      return true;
    }
    if (v1_later ? i1 : i2) return false;                    // the popping vertex must expand
    T = v1_later ? a.t : b.t; Tv = v1_later ? v1 : v2;
    // a face inside a cascade of c itself cannot update c (LabelStore::names) -- unless c is never fixed: an invalid vertex
    // pops without being fixed (:417-422) and keeps receiving updates from every face that fires later
    return (invalid && invalid[c]) || !names(T, c);
  }

  // event-ordered replay of the faces around c; win = corner record of the LAST accepted update (-1: none), with the
  // source distances and the candidate it was accepted with (the repulsive vector field is derived from it)
  // Faces that fire at the same pop (same popping vertex p = Tv; the two faces on either side of the edge (p, c) always
  // do) are visited in the order of the reference's neighbour loop (inflation_layer.cpp:423-427): p's edges in ascending
  // id, for each edge the lower-id face first; a face is reached through the first of its two edges at p.  The order
  // decides which of two exactly equal candidates is "accepted" (strict <, :297) -- i.e. the repulsive vector -- and the
  // heap key when only one of the faces has both sources inside the radius (:310).
  __device__ __forceinline__ uint32_t visit_key(uint32_t k, uint32_t p) const {
    const int4 ix = __ldg(&cor_idx[k]);
    const uint4 e = __ldg(&cor_eid[k]);
    const uint32_t k_ec = (e.x << 1) | ((uint32_t)ix.w & 1u);                       // edge(v1,v2) is at p either way
    const uint32_t k_pc = (uint32_t)ix.x == p ? ((e.y << 1) | (((uint32_t)ix.w >> 1) & 1u))    // p == v1: edge(v1,c)
                                              : ((e.z << 1) | (((uint32_t)ix.w >> 2) & 1u));   // p == v2: edge(v2,c)
    return k_ec < k_pc ? k_ec : k_pc;
  }
  // true if entry (T1, k1) precedes (T2, k2) in the reference's call order
  __device__ __forceinline__ bool fires_before(const EvTime& T1, uint32_t k1, uint32_t p1, const EvTime& T2, uint32_t k2, uint32_t p2) const {
    if (!teq(T1, T2)) return tless(T1, T2);
    if (p1 != p2) return k1 < k2;                            // (cannot happen: equal pop times name the same vertex)
    return visit_key(k1, p1) < visit_key(k2, p2);
  }

  // vertices with more than MAXF incident faces: repeated selection of the next face in call order by rescanning the
  // corner list (O(deg^2), rare) -- same rule as the buffered loop below
  __device__ __noinline__ void replay_big(uint32_t c, float band_end, uint32_t round, float& nd, EvFull& tc_out, int& win,
                                          float& wu1, float& wu2) const {
    const uint32_t kb = cor_ptr[c], ke = cor_ptr[c + 1];
    const float INF = __uint_as_float(INF_BITS);
    float cur = INF;
    EvFull tc = full_normal(INF, c);
    win = -1; wu1 = 0.0f; wu2 = 0.0f;
    const bool never_fixed = invalid && invalid[c];
    EvTime lastT = ev_normal(0.0f, 0); uint32_t lastK = 0, lastTv = 0; bool have_last = false;
    for (;;) {
      EvTime bT = lastT; float bu1 = 0, bu2 = 0; uint32_t bk = 0, bTv = 0; bool found = false;
      for (uint32_t k = kb; k < ke; ++k) {
        EvTime T; float u1, u2; uint32_t Tv;
        if (!corner_time(c, k, band_end, T, Tv, u1, u2)) continue;
        if (have_last && (k == lastK || !fires_before(lastT, lastK, lastTv, T, k, Tv))) continue;
        if (!found || fires_before(T, k, Tv, bT, bk, bTv)) { bT = T; bk = k; bTv = Tv; bu1 = u1; bu2 = u2; found = true; }
      }
      if (!found) break;
      if (!never_fixed && !less_T_full(bT, tc)) break;
      const float4 w = __ldg(&cor_wd[bk]);
      const float cand = inflation_candidate(bu1, bu2, w.z, w.y, w.x);
      if (cand < cur && backstep_ok(cand, bT, bTv, round)) {
        cur = cand; win = (int)bk; wu1 = bu1; wu2 = bu2;
        if (bu1 <= max_distance && bu2 <= max_distance) accept(c, cand, bT, tc);
      }
      lastT = bT; lastK = bk; lastTv = bTv; have_last = true;
    }
    nd = cur; tc_out = tc;
  }

  __device__ __forceinline__ void replay(uint32_t c, float band_end, uint32_t round, float& nd, EvFull& tc_out, int& win,
                                         float& wu1, float& wu2) const {
    const uint32_t kb = cor_ptr[c], ke = cor_ptr[c + 1];
    if (ke - kb > (uint32_t)MAXF) { replay_big(c, band_end, round, nd, tc_out, win, wu1, wu2); return; }
    EvTime Tt[MAXF]; float U1[MAXF], U2[MAXF]; uint32_t K[MAXF], TV[MAXF];
    int n = 0;
    for (uint32_t k = kb; k < ke && n < MAXF; ++k) {
      EvTime T; float u1, u2; uint32_t Tv;
      if (!corner_time(c, k, band_end, T, Tv, u1, u2)) continue;
      Tt[n] = T; U1[n] = u1; U2[n] = u2; K[n] = k; TV[n] = Tv; ++n;
    }
    const float INF = __uint_as_float(INF_BITS);
    float cur = INF;
    EvFull tc = full_normal(INF, c);                       // pop time = heap key; +inf while not inserted
    win = -1; wu1 = 0.0f; wu2 = 0.0f;
    // an invalid vertex is popped but never fixed (:417-422): it keeps receiving updates from every face
    const bool never_fixed = invalid && invalid[c];
    for (int i = 0; i < n; ++i) {
      int b = i;
      for (int j = i + 1; j < n; ++j)
        if (fires_before(Tt[j], K[j], TV[j], Tt[b], K[b], TV[b])) b = j;
      const EvTime T = Tt[b]; const float u1 = U1[b], u2 = U2[b]; const uint32_t k = K[b], Tv = TV[b];
      Tt[b] = Tt[i]; U1[b] = U1[i]; U2[b] = U2[i]; K[b] = K[i]; TV[b] = TV[i];
      if (!never_fixed && !less_T_full(T, tc)) break;      // c was popped (and fixed) before this face fires
      const float4 w = __ldg(&cor_wd[k]);
      const float cand = inflation_candidate(u1, u2, w.z, w.y, w.x);   // a = |v2c|, b = |v1c|, c = |v1v2|
#ifdef MNB_EMU_ACTIVE
      if (getenv("MNB_DBG_V") && c == (uint32_t)atoi(getenv("MNB_DBG_V"))) fprintf(stderr, "[r%u] c=%u face k=%u Tv=%u T=(%g,%u,%g,%g) u1=%g u2=%g cand=%g cur=%g tc=(%g,%u,%g) n=%d\n", round, c, k, Tv, T.a1, T.root, T.a2, T.a3, u1, u2, cand, cur, tc.t.a1, tc.t.root, tc.t.a2, n);
#endif
      if (cand < cur && backstep_ok(cand, T, Tv, round)) {                                    // :297 (non-finite candidates were mapped to +inf)
        cur = cand; win = (int)k; wu1 = u1; wu2 = u2;
        if (u1 <= max_distance && u2 <= max_distance) accept(c, cand, T, tc);   // :310 -> pq.insert(c, cand)
      }
    }
    nd = cur; tc_out = tc;
  }

  // Same collapse as CvpEllProblem::replay_sub8's fast path: if every firing face either is causal (candidate above its own
  // pop time) with both sources inside the radius (so the accepted value is also the heap key, :310), or fires after the
  // smallest causal candidate m, the call-ordered replay yields d = m and the pop time (m, c) -- no sorting of the faces,
  // no visit keys.  Returns false if the general replay is needed.
  __device__ __forceinline__ bool replay_fast(uint32_t c, float band_end, float& nd, EvTime& tc_out) const {
    const uint32_t kb = cor_ptr[c], ke = cor_ptr[c + 1];
    if (ke - kb > (uint32_t)MAXF || (invalid && invalid[c])) return false;
    const float INF = __uint_as_float(INF_BITS);
    float m = INF, tmin_nc = INF;                                       // smallest causal candidate / earliest non-causal face
    for (uint32_t k = kb; k < ke; ++k) {
      EvTime T; float u1, u2; uint32_t Tv;
      if (!corner_time(c, k, band_end, T, Tv, u1, u2)) continue;
      const float4 w = __ldg(&cor_wd[k]);
      const float cand = inflation_candidate(u1, u2, w.z, w.y, w.x);
      if (cand > T.a1) {                                               // causal
        if (!(u1 <= max_distance && u2 <= max_distance)) return false;   // accepted without (re)insertion: heap key != distance
        m = fminf(m, cand);
      } else {
        tmin_nc = fminf(tmin_nc, T.a1);
      }
    }
    if (__float_as_uint(tmin_nc) != INF_BITS && !(tmin_nc > m)) return false;   // a non-causal face that could fire before c pops
    nd = m; tc_out = ev_normal(m, c);
    return true;
  }

  __device__ __forceinline__ bool recompute(uint32_t c, float band_end, float /*goal*/, uint32_t round, const Label& old, float& nd, float& ntau) {
    EvTime tc; int win; float wu1, wu2;
    if (!replay_fast(c, band_end, nd, tc)) {   // (the collapse accepts no back-step: valid in strict rounds too)
      EvFull tf;
      replay(c, band_end, round, nd, tf, win, wu1, wu2);
      tc = finish(tf, old.t);
    }
    ntau = tc.a1;
    if (__float_as_uint(nd) == __float_as_uint(old.d) && teq(tc, old.t)) return false;
    store_label(c, nd, tc, __float_as_uint(old.d) != INF_BITS, round);
    return true;
  }
};

// ---------------------------------------------------------------------------
// Dijkstra: d[c] = min over expandable neighbours u of fl(d[u] + w(u,c));
// among equal sums the neighbour that pops first wins (strict '<' at
// dijkstra_mesh_planner.cpp:332): order (d[u], u).  Edge weights are >= 0 so a
// vertex always pops at its own key: tau = d, one level.
//   adj_nw[k] = {neighbour id, float bits of the edge weight}
// The label word S is the engine's uint4 {d, tau, -, -} or, in the lean workspace of the batch kernel
// (k_dijkstra_batch), the float d alone: tau = d carries no information of its own.
// pred may be null: no predecessors are written.
// ---------------------------------------------------------------------------
template <class S>
struct DijkstraProblemT : TimeAlg {
  static constexpr bool HAS_GOAL_TIME = false;    // edge weights >= 0: vertices pop in potential order, the test on the value is exact
  static constexpr bool CAN_SKIP = false;
  const uint32_t* __restrict__ adj_ptr;
  const uint2* __restrict__ adj_nw;
  const float* __restrict__ cost;
  const uint8_t* __restrict__ invalid;  // may be null
  S* state;
  uint32_t* pred;
  double cost_limit;
  float deferred_m;                     // unused (edge weights >= 0: no back-steps), kept for the engine interface
  int strict;

  __device__ __forceinline__ static float label_d(const uint4& s) { return __uint_as_float(s.x); }
  __device__ __forceinline__ static float label_d(float s) { return s; }
  __device__ __forceinline__ static float label_tau(const uint4& s) { return __uint_as_float(s.y); }
  __device__ __forceinline__ static float label_tau(float s) { return s; }
  __device__ __forceinline__ void store_d(uint32_t c, float d) const {
    if constexpr (std::is_same<S, float>::value) __stcg(&state[c], d);
    else __stcg(&state[c], make_uint4(__float_as_uint(d), __float_as_uint(d), 0u, 0u));
  }
  __device__ __forceinline__ Label load_label(uint32_t v) const {
    const S s = __ldcg(&state[v]);
    Label l; l.d = label_d(s); l.t = ev_normal(label_tau(s), v);
    return l;
  }
  __device__ __forceinline__ bool eligible(uint32_t x) const { return !(invalid && invalid[x]); }  // :328
  __device__ __forceinline__ static bool never_fixed(uint32_t) { return false; }

  template <class F>
  __device__ __forceinline__ void activate(uint32_t c, F push) const {
    const uint32_t kb = adj_ptr[c], ke = adj_ptr[c + 1];
    for (uint32_t k = kb; k < ke; ++k) push(__ldg(&adj_nw[k]).x);
  }

  __device__ __forceinline__ bool recompute(uint32_t c, float band_end, float goal, uint32_t /*round*/, const Label& old, float& nd, float& ntau) {
    const uint32_t kb = adj_ptr[c], ke = adj_ptr[c + 1];
    float best = __uint_as_float(INF_BITS), best_du = best; uint32_t best_u = c;
    for (uint32_t k = kb; k < ke; ++k) {
      const uint2 nw = __ldg(&adj_nw[k]);
      const uint32_t u = nw.x;
      const float du = label_d(__ldcg(&state[u]));
      if (!(du < band_end)) continue;
      if (du > goal) continue;                               // :299
      if ((double)__ldg(&cost[u]) > cost_limit) continue;    // :302
      const float tmp = __fadd_rn(du, __uint_as_float(nw.y)); // :331
      if (tmp < best || (tmp == best && __float_as_uint(tmp) != INF_BITS &&
                         (du < best_du || (du == best_du && u < best_u)))) {
        best = tmp; best_du = du; best_u = u;
      }
    }
    nd = best; ntau = best;
    if (__float_as_uint(nd) == __float_as_uint(old.d)) {
      // same potential; the predecessor can still change among exact ties
      if (pred && __float_as_uint(nd) != INF_BITS && pred[c] != best_u) pred[c] = best_u;
      return false;
    }
    store_d(c, nd);
    if (pred) pred[c] = best_u;
    return true;
  }
};
using DijkstraProblem = DijkstraProblemT<uint4>;

// ---------------------------------------------------------------------------
// Dijkstra field repair (k_dijkstra_batch_repair): the same pull on the caller's rows, which hold realizable upper bounds
// of the new distances from the start.  A band-filtered pull can miss a source beyond the band, so a label never rises:
// the smaller of the stored and the pulled value stays (in a fresh wave the two are always equal).  The round loop
// activates on a change of label (REPAIR) and logs every vertex it marks in log[*log_n++] so that the kernel can reset
// the marks of the wave without a V-sized pass.
// ---------------------------------------------------------------------------
struct DijkstraRepairProblem : DijkstraProblemT<float> {
  static constexpr bool REPAIR = true;
  uint32_t* log;
  unsigned int* log_n;

  __device__ __forceinline__ void log_mark(uint32_t x) const { log[atomicAdd(log_n, 1u)] = x; }

  __device__ __forceinline__ bool recompute(uint32_t c, float band_end, float /*goal*/, uint32_t /*round*/, const Label& old, float& nd, float& ntau) {
    const uint32_t kb = adj_ptr[c], ke = adj_ptr[c + 1];
    float best = __uint_as_float(INF_BITS), best_du = best; uint32_t best_u = c;
    for (uint32_t k = kb; k < ke; ++k) {
      const uint2 nw = __ldg(&adj_nw[k]);
      const uint32_t u = nw.x;
      const float du = __ldcg(&state[u]);
      if (!(du < band_end)) continue;
      if ((double)__ldg(&cost[u]) > cost_limit) continue;
      const float tmp = __fadd_rn(du, __uint_as_float(nw.y));
      if (tmp < best || (tmp == best && __float_as_uint(tmp) != INF_BITS &&
                         (du < best_du || (du == best_du && u < best_u)))) {
        best = tmp; best_du = du; best_u = u;
      }
    }
    if (!(best < old.d)) {                 // no better path: the stored label (and, unless tied, its predecessor) stays
      nd = old.d; ntau = old.d;
      if (best == old.d && __float_as_uint(best) != INF_BITS && pred[c] != best_u) pred[c] = best_u;
      return false;
    }
    nd = best; ntau = best;
    store_d(c, nd);
    pred[c] = best_u;
    return true;
  }
};


// ---------------------------------------------------------------------------
// Dijkstra, 8 lanes per candidate: the adjacency lives in an ELL table, row c = 8 slots x {neighbour, weight bits,
// -, degree} (one 128-byte line), each lane relaxes one edge and the lexicographic argmin (tmp, du, u) -- the
// reference's strict `<` in pop order (dijkstra:331-335) -- is taken with three shuffle steps.  Vertices with more
// than 8 neighbours take the CSR loop on lane 0.
// ---------------------------------------------------------------------------
struct DijkstraEllProblem : DijkstraProblem {
  static constexpr bool TWO_SOURCES = false;
  static constexpr bool PLAIN_FAST = false;
  static constexpr bool prefetch_marks = true;
  const uint4* __restrict__ ell_adj;
  uint32_t* ver;

  __device__ __forceinline__ int4 load_row_idx(uint32_t c, uint32_t j) const {
    const uint4 r = __ldg(&ell_adj[(size_t)c * ELL_W + j]);
    return make_int4((int)r.x, (int)r.y, 0, (int)r.w);            // {neighbour or -1, weight bits, -, degree}
  }
  __device__ __forceinline__ float4 load_row_w(uint32_t, uint32_t) const { return make_float4(0.f, 0.f, 0.f, 0.f); }
  __device__ __forceinline__ uint4 pack_label(uint32_t, float d, const EvTime& t) const {
    return make_uint4(__float_as_uint(d), __float_as_uint(t.a1), 0u, 0u);
  }
  __device__ __forceinline__ Label unpack_label(uint32_t v, const uint4& s) const {
    Label l; l.d = __uint_as_float(s.x); l.t = ev_normal(__uint_as_float(s.y), v);
    return l;
  }
  __device__ __forceinline__ void store_label(uint32_t c, float d, const EvTime& t, bool, uint32_t) const {
    __stcg(&state[c], make_uint4(__float_as_uint(d), __float_as_uint(t.a1), 0u, 0u));
  }
  // one relaxation candidate of the argmin; returns true if (tmp, du, u) precedes (best, best_du, best_u)
  __device__ __forceinline__ static bool better(float tmp, float du, uint32_t u, float best, float best_du, uint32_t best_u) {
    return tmp < best || (tmp == best && __float_as_uint(tmp) != INF_BITS && (du < best_du || (du == best_du && u < best_u)));
  }
  __device__ __noinline__ void replay_serial(uint32_t c, float band_end, float goal, float& best, uint32_t& best_u) const {
    const uint32_t kb = adj_ptr[c], ke = adj_ptr[c + 1];
    best = __uint_as_float(INF_BITS); float best_du = best; best_u = c;
    for (uint32_t k = kb; k < ke; ++k) {
      const uint2 nw = __ldg(&adj_nw[k]);
      const uint32_t u = nw.x;
      const float du = __uint_as_float(__ldcg(&state[u]).x);
      if (!(du < band_end) || du > goal || (double)__ldg(&cost[u]) > cost_limit) continue;     // :299, :302
      const float tmp = __fadd_rn(du, __uint_as_float(nw.y));                                   // :331
      if (better(tmp, du, u, best, best_du, best_u)) { best = tmp; best_du = du; best_u = u; }
    }
  }
  __device__ __forceinline__ void replay_sub8(uint32_t c, uint32_t j, bool has, const int4& ix, const float4&, float band_end,
                                              float goal, uint32_t /*round*/, const uint32_t* mark, const EvTime& /*old_t*/, float& nd, EvTime& nt, int& deg_out,
                                              uint32_t& mk1, uint32_t& mk2) const {
    constexpr unsigned FULL = 0xffffffffu;
    const float INF = __uint_as_float(INF_BITS);
    const int deg = __shfl_sync(FULL, ix.w, 0, 8);
    deg_out = deg;
    const bool big = has && deg > (int)ELL_W;
    float tmp = INF, du = INF; uint32_t u = 0xffffffffu;
    if (has && !big && ix.x != ELL_EMPTY) {
      u = (uint32_t)ix.x;
      du = __uint_as_float(__ldcg(reinterpret_cast<const uint32_t*>(state) + 4 * (size_t)u));
      mk1 = __ldcg(&mark[u]);
      const float cu = __ldg(&cost[u]);
      if (du < band_end && !(du > goal) && !((double)cu > cost_limit))                         // :299, :302
        tmp = __fadd_rn(du, __int_as_float(ix.y));                                             // :331
      else du = INF;
    }
    mk2 = MARK_FIXED;
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) {
      const float ot = __shfl_xor_sync(FULL, tmp, o, 8), od = __shfl_xor_sync(FULL, du, o, 8);
      const uint32_t ou = __shfl_xor_sync(FULL, u, o, 8);
      if (better(ot, od, ou, tmp, du, u)) { tmp = ot; du = od; u = ou; }
    }
    if (big && j == 0) { float ts; uint32_t us; replay_serial(c, band_end, goal, ts, us); tmp = ts; u = us; }   // (address-taken copies stay in the rare branch)
    if (__ballot_sync(FULL, big)) { tmp = __shfl_sync(FULL, tmp, 0, 8); u = __shfl_sync(FULL, u, 0, 8); }
    nd = tmp; nt = ev_normal(tmp, c);
    // predecessor of the winning relaxation (it can change among exact ties without the potential changing)
    // (a label can also fall back to +inf when the goal cutoff removes its sources: predecessor = self, dijkstra:269)
    if (has && j == 0) pred[c] = __float_as_uint(tmp) != INF_BITS ? u : c;
  }
};

}  // namespace mnb
