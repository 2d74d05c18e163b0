// Lean round loop for BATCHES of full-field CVP plans (mnb_cvp_batch): one wavefront per CTA / cluster, hundreds in flight.
//
// Same algorithm, same label format and bit-identical results as run_band_rounds_sub8 (band_engine.cuh); what differs is
// what the hot loop carries.  The generic loop serves single plans (goal cutoff + re-queueing, in-round sweeps, robot
// bookkeeping) and holds the whole problem object live: at the 64 registers a 2-CTA/SM batch
// kernel may use it spilled: a large share of the executed instructions become local loads and stores, and with
// hundreds of wavefronts in flight the local-memory footprint does not fit the L2.  A batch needs none of the extras:
//   * fast path (98 % of the evaluations): every source label is plain (one level), no source can be a seed, the causal
//     collapse applies -> the new label is min over the causal faces; nothing but the kernel parameters (constant bank)
//     and five per-wavefront pointers stay live, no problem object, no pop-time algebra;
//   * anything else (cascade members among the sources, a possible seed, non-causal faces that may fire first, more than
//     8 faces, strict rounds) -> the warp calls the generic CvpEllProblem::replay_sub8 through a __noinline__ wrapper
//     that builds the problem object on its own stack frame;
//   * the "has activated its neighbours" state travels in bit 31 of the list entry (no mark[] load per evaluation);
//     stage pushes are warp-aggregated by hand (one shared atomic per warp and kind).
#pragma once
#include "problems.cuh"

namespace mnb {

constexpr uint32_t LIST_ACTIVATED = 0x80000000u;

struct BatchGroup {          // per-wavefront pointers (group g of the workspace)
  uint4* state; uint32_t* root_arr; uint32_t* ext_arr; uint32_t* chg; uint32_t* mark; uint32_t* pool; uint32_t pool_cap; GroupCtl* ctl;
  uint4* skipw;             // clean-candidate words {relevant re-label of a neighbour: even rounds, odd rounds, band-excluded source, -}
};

template <class Args>
__device__ __forceinline__ void batch_make_problem(const Args& a, const BatchGroup& G, const SeedFace& sd, int strict,
                                                   CvpEllProblem& prob) {
  cvp_ell_problem(a, G.state, G.ext_arr, G.root_arr, G.chg, G.pool, G.pool_cap, G.ctl, sd, ev_normal(__uint_as_float(INF_BITS), 0u), false, prob);
  prob.strict = strict;
}

// the generic 8-lane evaluation (every lane of the warp calls this; groups that do not need it pass has = false)
template <class Args>
__device__ __noinline__ void batch_slow_eval(const Args& a, const BatchGroup& G, const SeedFace& sd, int strict, uint32_t c, uint32_t j,
                                             bool has, const int4& ix, const float4& w, float band_end, uint32_t round, const uint4& old_bits,
                                             float& nd, EvTime& nt, float& deferred_m) {
  CvpEllProblem prob;
  batch_make_problem(a, G, sd, strict, prob);
  const Label old = has ? prob.unpack_label(c, old_bits) : prob.unpack_label(0u, state_inf());
  int deg; uint32_t mk1 = MARK_FIXED, mk2 = MARK_FIXED;
  prob.replay_sub8(c, j, has, ix, w, band_end, __uint_as_float(INF_BITS), round, G.mark, old.t, nd, nt, deg, mk1, mk2);
  deferred_m = prob.deferred_m;
}

// store of a label that is not plain (cascade member): compares with the old label, returns "changed"
template <class Args>
__device__ __noinline__ bool batch_store_general(const Args& a, const BatchGroup& G, const SeedFace& sd, uint32_t c, uint32_t j, bool has,
                                                 const uint4& old_bits, float nd, const EvTime& nt, uint32_t round) {
  if (!has) return false;
  CvpEllProblem prob;
  batch_make_problem(a, G, sd, 0, prob);
  const Label old = prob.unpack_label(c, old_bits);
  const bool changed = __float_as_uint(nd) != old_bits.x || !prob.teq(nt, old.t);
  if (changed && j == 0) prob.store_label(c, nd, nt, old_bits.x != INF_BITS, round);
  return changed;
}

// the batch kernels stage a whole round of a 1M-vertex plan (~3.5 k candidates + activations) in shared memory
using BatchStage = StageT<6144>;
__device__ __forceinline__ void batch_stage_write(BatchStage& st, unsigned int slot, uint32_t v, uint32_t* list_next, unsigned int* count_next) {
  if (slot < (unsigned)BatchStage::CAP) st.buf[slot] = v;
  else list_next[atomicAdd(count_next, 1u)] = v;     // overflow: straight to global
}

// vertices with more than 8 faces: neighbours beyond the ELL row are activated through the CSR corner list (rare)
template <class Args>
__device__ __noinline__ void batch_activate_big(const Args& a, const BatchGroup& G, uint32_t c, BatchStage& st, uint32_t* list_next, unsigned int* count_next) {
  const uint32_t kb = a.cor_ptr[c], ke = a.cor_ptr[c + 1];
  for (uint32_t k = kb; k < ke; ++k) {
    const int4 ix = __ldg(&a.cor_idx[k]);
    const uint32_t xs[2] = {(uint32_t)ix.x, (uint32_t)ix.y};
    for (int t = 0; t < 2; ++t) {
      const uint32_t x = xs[t];
      if (__ldcg(&G.mark[x]) != MARK_NONE) continue;
      if (a.invalid && a.invalid[x]) continue;
      if ((double)a.cost[x] >= a.cost_limit) continue;
      if (atomicCAS(&G.mark[x], MARK_NONE, MARK_CAND) == MARK_NONE) batch_stage_write(st, atomicAdd(&st.n, 1u), x, list_next, count_next);
    }
  }
}

// vertices with more than 8 faces: the face neighbours beyond the ELL row are told about a re-label through the CSR list
template <class Args>
__device__ __noinline__ void batch_notify_big(const Args& a, const BatchGroup& G, uint32_t c, uint32_t buf, uint32_t key_bits) {
  const uint32_t kb = a.cor_ptr[c], ke = a.cor_ptr[c + 1];
  for (uint32_t k = kb; k < ke; ++k) {
    const int4 ix = __ldg(&a.cor_idx[k]);
    atomicMin(reinterpret_cast<uint32_t*>(G.skipw) + 4 * (size_t)(uint32_t)ix.x + buf, key_bits);
    atomicMin(reinterpret_cast<uint32_t*>(G.skipw) + 4 * (size_t)(uint32_t)ix.y + buf, key_bits);
  }
}

// Work queue of a CTA: the candidates of the current chunk that have to be evaluated (phase B below)
struct BatchWork { static constexpr int CAP = 2048; uint32_t q[CAP]; uint32_t sq[CAP]; unsigned int n, ns; };

// Phase C of a round (see run_band_rounds_batch): 8 lanes per candidate, the general evaluation -- cascade members among
// the sources, possible seeds, non-causal faces that may fire first, more than 8 faces, strict rounds.  A few percent of
// the evaluations; kept out of line so that its register needs do not weigh on the throughput phases.
template <class Args>
__device__ __noinline__ void batch_general_phase(const Args& a, const BatchGroup& G, const SeedFace& sd, BatchStage& st, BatchWork& wk,
                                                 uint32_t* list_n, unsigned int* count_next, const float band_end, const int strict, const uint32_t r,
                                                 float& my_mtau_io, float& my_lo_io, unsigned int& my_recomputes_io) {
  constexpr unsigned FULL = 0xffffffffu;
  const float INF = __uint_as_float(INF_BITS);
  GroupCtl* const ctl = G.ctl; (void)ctl;
  uint32_t* const skw = reinterpret_cast<uint32_t*>(G.skipw);
  const uint32_t lane = threadIdx.x & 31, j = lane & 7, sh = lane & ~7u;
  const uint32_t lt = (1u << lane) - 1u;
  const uint32_t buf_now = r & 1u;
  float my_mtau = my_mtau_io, my_lo = my_lo_io; unsigned int my_recomputes = my_recomputes_io;
  const unsigned int nw = wk.ns;
      for (unsigned int qb = (threadIdx.x >> 5) * 4u; qb < nw; qb += (blockDim.x >> 3)) {
      const unsigned int q = qb + (lane >> 3);
      const bool has = q < nw;
      const uint32_t ce = has ? wk.sq[q] : 0u;
      const uint32_t c = ce & ~LIST_ACTIVATED;
      const bool activated = (ce & LIST_ACTIVATED) != 0u;
      const uint4 ob = __ldcg(&G.state[c]);
      const int4 ix = __ldg(&a.ell_idx[(size_t)c * ELL_W + j]);
      const float4 w = __ldg(&a.ell_w[(size_t)c * ELL_W + j]);
      const float tau = __uint_as_float(ob.y);
      const int deg = __shfl_sync(FULL, ix.w, 0, 8);
      bool valid = has && deg <= (int)ELL_W && ix.x != ELL_EMPTY;
      bool slow = has && (deg > (int)ELL_W || strict);
      float T1 = INF, excl = INF;                      // excl: smallest finite source label of this lane's face beyond the band end
      double U = 0.0, X = 0.0;
      if (!__any_sync(FULL, has)) continue;
      if (valid) {
        const uint32_t v1 = (uint32_t)ix.x, v2 = (uint32_t)ix.y;
        const uint4 sa = __ldcg(&G.state[v1]), sb = __ldcg(&G.state[v2]);
        const double2* gp = reinterpret_cast<const double2*>(a.ell_geo) + 2 * ((size_t)c * ELL_W + j);
        const double2 g01 = __ldg(gp), g23 = __ldg(gp + 1);
        const float da = __uint_as_float(sa.x), db = __uint_as_float(sb.x);
        if ((sa.z | sa.w | sb.z | sb.w) >> 31) slow = true;             // a cascade member among the sources: general order
        if (da <= sd.seed_max || db <= sd.seed_max) slow = true;        // possibly a seed (fixed before it pops): general rule
        if (a.invalid && (a.invalid[v1] || a.invalid[v2])) valid = false;
        if (sa.x != INF_BITS && !(da < band_end)) excl = da;
        if (sb.x != INF_BITS && !(db < band_end)) excl = fminf(excl, db);
        if (!(da < band_end) || !(db < band_end)) valid = false;
        if (valid) {
          // plain labels pop at (key, id); the face fires at the later of the two
          const float ta = __uint_as_float(sa.y), tb = __uint_as_float(sb.y);
          const bool v1_later = tb < ta || (tb == ta && v2 < v1);
          T1 = v1_later ? ta : tb;
          CvpEllProblem::FaceGeo fg; fg.p = g01.x; fg.hc = g01.y; fg.t0a = g23.x;
          CvpEllProblem::eval_face_geo((double)da, (double)db, (double)w.z, (double)w.y, (double)w.x, fg, U, X);
        }
      }
      // causal collapse (CvpEllProblem::replay_sub8): d = min over the causal faces if no other face can fire before it
      const float Xf = (float)X;
      const bool causal = valid && Xf > T1 && U <= X;
      float m = causal ? Xf : INF;
#pragma unroll
      for (int o = 4; o > 0; o >>= 1) m = fminf(m, __shfl_xor_sync(FULL, m, o, 8));
      if (valid && !causal && !(T1 > m)) slow = true;
      float nd = m, nt_a1 = m;
      bool plain_new = true;
      EvTime nt = ev_normal(m, c);
      const unsigned slow_mask = __ballot_sync(FULL, slow);
      if (slow_mask) {                                                   // (warp-uniform branch)
        const bool gslow = ((slow_mask >> sh) & 0xFFu) != 0u;            // my 8-lane group needs the general evaluation
        float snd, dm; EvTime snt;
        batch_slow_eval(a, G, sd, strict, c, j, has && gslow, ix, w, band_end, r, ob, snd, snt, dm);
        if (gslow) {
          nd = snd; nt = snt; nt_a1 = snt.a1;
          plain_new = snt.a2 == 0.0f && snt.root == c;
          my_mtau = fminf(my_mtau, dm);                                  // deferred back-steps are pending changes
        }
      }
      bool changed;
      if (plain_new) {
        const uint4 nb = make_uint4(__float_as_uint(nd), __float_as_uint(nt_a1), 0u, 0u);
        changed = has && (ob.x != nb.x || ob.y != nb.y || ob.z != 0u || ob.w != 0u);
        if (changed && j == 0) {
          if (ob.x != INF_BITS) __stcg(&G.chg[c], r + 1u);
          __stcg(&G.state[c], nb);
        }
      } else {
        changed = batch_store_general(a, G, sd, c, j, has, ob, nd, nt, r);
      }
      const bool act_now = has && !activated && __float_as_uint(nd) != INF_BITS;
      const bool lead = has && j == 0;
      {
        // clean-candidate bookkeeping (see the header of this function).  A source beyond the band end matters only if its
        // face could fire before c pops: the face time's first level is >= the source's label.  The general path and
        // vertices with more than 8 faces are not tracked per source: they are re-evaluated every round (excl = 0).
        float e = (excl <= nt_a1) ? excl : INF;
#pragma unroll
        for (int o = 4; o > 0; o >>= 1) e = fminf(e, __shfl_xor_sync(FULL, e, o, 8));
        const bool untracked = deg > (int)ELL_W || (slow_mask && ((slow_mask >> sh) & 0xFFu));
        if (lead) __stcg(&skw[4 * (size_t)c + 2], untracked ? 0u : __float_as_uint(e));
        if (changed) {
          // tell the vertices that read c's label (its face neighbours): smallest pop-time key involved in the re-label
          const uint32_t kb = __float_as_uint(fminf(tau, nt_a1));
          if (deg <= (int)ELL_W && ix.x != ELL_EMPTY) {
            atomicMin(&skw[4 * (size_t)(uint32_t)ix.x + buf_now], kb);
            atomicMin(&skw[4 * (size_t)(uint32_t)ix.y + buf_now], kb);
          }
          if (j == 0 && deg > (int)ELL_W) batch_notify_big(a, G, c, buf_now, kb);
        }
      }
#ifdef MNB_EMU_ACTIVE   // evaluation statistics on the CPU interpreter (tests/emu): what the recomputes of a batch are spent on
      if (lead) atomicAdd(&ctl->t_ph[__float_as_uint(nd) == INF_BITS ? 0 : (changed ? 1 : 2)], 1ull);
      if (lead && slow_mask && ((slow_mask >> sh) & 0xFFu)) atomicAdd(&ctl->t_ph[3], 1ull);
#endif
      if (lead) {
        my_recomputes++;
        if (changed) my_mtau = fminf(my_mtau, fminf(tau, nt_a1));
        my_lo = fminf(my_lo, nt_a1);                                     // smallest pop time still in flight: the band follows it
      }
      {   // the candidate survives into the next round's list (one shared atomic per warp)
        const unsigned pm = __ballot_sync(FULL, lead);
        unsigned int base = 0;
        if (lane == (unsigned)(__ffs(pm) - 1)) base = atomicAdd(&st.n, (unsigned)__popc(pm));
        base = __shfl_sync(FULL, base, (__ffs(pm) - 1) & 31);
        if (lead) batch_stage_write(st, base + __popc(pm & lt), c | ((activated || act_now) ? LIST_ACTIVATED : 0u), list_n, count_next);
      }
      if (__any_sync(FULL, act_now)) {
        // a vertex that holds a finite label pulls its neighbours into the candidate set (once): every lane offers the two
        // source vertices of its own corner
        bool p1 = false, p2 = false;
        if (act_now && deg <= (int)ELL_W && ix.x != ELL_EMPTY) {
          const uint32_t x1 = (uint32_t)ix.x, x2 = (uint32_t)ix.y;
          if (__ldcg(&G.mark[x1]) == MARK_NONE && !(a.invalid && a.invalid[x1]) && !((double)__ldg(&a.cost[x1]) >= a.cost_limit))
            p1 = atomicCAS(&G.mark[x1], MARK_NONE, MARK_CAND) == MARK_NONE;
          if (__ldcg(&G.mark[x2]) == MARK_NONE && !(a.invalid && a.invalid[x2]) && !((double)__ldg(&a.cost[x2]) >= a.cost_limit))
            p2 = atomicCAS(&G.mark[x2], MARK_NONE, MARK_CAND) == MARK_NONE;
        }
        const unsigned b1 = __ballot_sync(FULL, p1), b2 = __ballot_sync(FULL, p2);
        const unsigned tot = (unsigned)(__popc(b1) + __popc(b2));
        if (tot) {
          const unsigned int base = warp_reserve(&st.n, tot);
          if (p1) batch_stage_write(st, base + __popc(b1 & lt), (uint32_t)ix.x, list_n, count_next);
          if (p2) batch_stage_write(st, base + __popc(b1) + __popc(b2 & lt), (uint32_t)ix.y, list_n, count_next);
        }
        if (act_now && j == 0 && deg > (int)ELL_W) batch_activate_big(a, G, c, st, list_n, count_next);
      }
      }   // phase C
  my_mtau_io = my_mtau; my_lo_io = my_lo; my_recomputes_io = my_recomputes;
}


// Preconditions as for run_band_rounds (band_engine.cuh); list entries of list0 carry no flag bits; skipw = {inf, inf, 0, 0}.
//
// A round has two phases per chunk of the CTA's share of the candidate list:
//   A (one THREAD per candidate): settled?  clean?  A candidate is CLEAN -- its label cannot change, it is carried over
//     without being evaluated -- if (1) no face neighbour was re-labelled during the previous round with a pop time that
//     is not above the candidate's own (a face fires at or after the pop of its later source: a source that pops after
//     the candidate, before and after its re-label, cannot reach it), and (2) no source that lay beyond the band end at
//     the candidate's last evaluation has come inside since.  (1) is a per-vertex float "smallest relevant re-label"
//     that neighbours lower with fire-and-forget atomicMin, double-buffered by round parity so that it is only ever read
//     across the round barrier; (2) is one float per vertex written by its own last evaluation.  On the terrain 64 % of
//     the evaluations of the plain round loop find nothing changed; this phase costs them ~25 thread-instructions.
//   B (8 lanes per candidate): the evaluation proper, on the compacted work queue.
// TARGETS (matrix form): the loop ends once every target of a.tg has settled, as in run_band_rounds.  STOP_ON_OVERFLOW
// (the batch replan): the loop also ends once the level pool has overflowed, as the resumed single plan's does.
template <int CS, bool TARGETS = false, bool STOP_ON_OVERFLOW = false, class Args>
__device__ __forceinline__ void run_band_rounds_batch(const Args& a, const BatchGroup& G, uint32_t* list0, uint32_t* list1, BatchStage& st,
                                                      BatchWork& wk, const float delta, const uint32_t gthreads, const uint32_t gtid,
                                                      const SeedFace& sd, const float band_end_init) {
  constexpr unsigned FULL = 0xffffffffu;
  const float INF = __uint_as_float(INF_BITS);
  GroupCtl* const ctl = G.ctl;
  uint32_t* const skw = reinterpret_cast<uint32_t*>(G.skipw);
  const uint32_t lane = threadIdx.x & 31, j = lane & 7, sh = lane & ~7u;
  const uint32_t lt = (1u << lane) - 1u;
  const uint32_t nblk = gthreads / blockDim.x, blk = gtid / blockDim.x;
  float band_end_prev = band_end_init;
  unsigned int my_recomputes = 0, my_settled = 0, my_skipped = 0;     // per round (flushed to the 64-bit counters at its end)
  float lo_best = -1.0f; int stagnant = 0, strict = 0;
  uint32_t r = 0;
  for (;; ++r) {
    const uint32_t slot = r % 3, prev = (r + 2) % 3, next = (r + 1) % 3;
    const unsigned int n = __ldcg(&ctl->count[slot]);
    const float m_prev = __uint_as_float(__ldcg(&ctl->m_tau[prev]));
    const float lo_prev = __uint_as_float(__ldcg(&ctl->lo[prev]));
    const unsigned int stop = __ldcg(&ctl->stop_ring[r & 1]);
    if (n == 0 || stop || r > a.max_rounds) break;           // r is group-uniform: the watchdog cannot deadlock the barrier
    if constexpr (TARGETS) if (__ldcg(&ctl->done_ring[r & 1])) break;     // every target has settled (see run_band_rounds)
    if (r > 0 && __float_as_uint(m_prev) == INF_BITS && __float_as_uint(lo_prev) == INF_BITS) break;
    // stagnation watch (see run_band_rounds): labels keep changing but the earliest unsettled pop time does not move
    if (r > 0 && __float_as_uint(m_prev) != INF_BITS && !(lo_prev > lo_best)) { if (++stagnant >= STAGNATION_ROUNDS) strict = 1; }
    else { stagnant = 0; if (lo_prev > lo_best) lo_best = lo_prev; }
    float band_end = lo_prev + delta;
    if (!(band_end > band_end_prev)) band_end = band_end_prev;
    const uint32_t* list_r = (r & 1) ? list1 : list0;
    uint32_t* list_n = (r & 1) ? list0 : list1;
    unsigned int* const count_next = &ctl->count[next];
    band_advance<false, STOP_ON_OVERFLOW>(ctl, gtid, r, INF_BITS, stop, a.cancel_flag);
    const uint32_t buf_now = r & 1u, buf_prev = buf_now ^ 1u;      // re-labels of this round / of the previous round
    float my_mtau = INF, my_lo = INF;
    const unsigned int cnt = n > blk ? (n - blk + nblk - 1) / nblk : 0u;
    for (unsigned int cb = 0; cb < cnt; cb += (unsigned)BatchWork::CAP) {
      const unsigned int ce_end = min(cnt, cb + (unsigned)BatchWork::CAP);
      // ---------------- phase A: one thread per candidate ----------------
      for (unsigned int ib = cb + (threadIdx.x & ~31u); ib < ce_end; ib += blockDim.x) {
        const unsigned int i = ib + lane;
        const bool has = i < ce_end;
        uint32_t ce = 0u; float tau = 0.0f; bool settled = false, clean = false;
        if (has) {
          ce = __ldcg(&list_r[(size_t)i * nblk + blk]);
          const uint32_t c = ce & ~LIST_ACTIVATED;
          tau = __uint_as_float(__ldcg(reinterpret_cast<const uint32_t*>(G.state) + 4 * (size_t)c + 1));
          settled = tau < m_prev && tau < band_end_prev;   // converged prefix: the sequential algorithm has popped c with this label
          if constexpr (TARGETS) if (settled) settle_target(ctl, a.tg.bits, c, r);
          if (!settled) {
            const uint4 sk = __ldcg(&G.skipw[c]);
            const uint32_t dmb = buf_prev ? sk.y : sk.x;
            if (dmb != INF_BITS) __stcg(&skw[4 * (size_t)c + buf_prev], INF_BITS);      // consumed (nobody writes this buffer during this round)
            clean = !strict && !(__uint_as_float(dmb) <= tau) && !(band_end > __uint_as_float(sk.z));
          }
        }
        if (settled) my_settled++;
        const bool keep = has && !settled && clean, work = has && !settled && !clean;
        if (keep) { my_skipped++; my_lo = fminf(my_lo, tau); }
        const unsigned km = __ballot_sync(FULL, keep), wm = __ballot_sync(FULL, work);
        if (km) {
          const unsigned int base = warp_reserve(&st.n, (unsigned)__popc(km));
          if (keep) batch_stage_write(st, base + __popc(km & lt), ce, list_n, count_next);
        }
        if (wm) {
          const unsigned int base = warp_reserve(&wk.n, (unsigned)__popc(wm));
          if (work) wk.q[base + __popc(wm & lt)] = ce;
        }
      }
      __syncthreads();
      const unsigned int nwork = wk.n;
      // ---------------- phase B: one THREAD per candidate, plain causal evaluations only ----------------
      // The throughput form of the evaluation (CvpEllProblem::eval_plain): a thread walks the faces of its candidate (ELL
      // row), every source label plain, no possible seed, and the causal collapse applies: d = min over the causal faces.
      // ~25 warp-instructions per candidate instead of ~140 for the 8-lane form, 32 candidates per warp in flight.  Anything
      // else is deferred to phase C.
      for (unsigned int ib = (threadIdx.x & ~31u); ib < nwork; ib += blockDim.x) {
        const unsigned int i = ib + lane;
        const bool has = i < nwork;
        bool defer = false;
        uint32_t ce = 0u, c = 0u; uint4 ob = make_uint4(0u, 0u, 0u, 0u);
        float m = INF, excl = INF;
        if (has) {
          ce = wk.q[i]; c = ce & ~LIST_ACTIVATED;
          ob = __ldcg(&G.state[c]);
          defer = strict || !CvpEllProblem::eval_plain(a.ell_idx, a.ell_w, a.ell_geo, a.invalid, G.state, sd.seed_max, band_end, c, m, excl);
        }
        const bool done = has && !defer;
        bool changed = false, act_now = false;
        if (done) {
          const float tau = __uint_as_float(ob.y);
          const uint32_t mb = __float_as_uint(m);
          changed = ob.x != mb || ob.y != mb || ob.z != 0u || ob.w != 0u;
          if (changed) {
            if (ob.x != INF_BITS) __stcg(&G.chg[c], r + 1u);
            __stcg(&G.state[c], make_uint4(mb, mb, 0u, 0u));
            my_mtau = fminf(my_mtau, fminf(tau, m));
          }
          __stcg(&skw[4 * (size_t)c + 2], __float_as_uint(excl <= m ? excl : INF));
          my_recomputes++;
          my_lo = fminf(my_lo, m);
          act_now = !(ce & LIST_ACTIVATED) && mb != INF_BITS;
          if (changed || act_now) {
            // tell the face neighbours about the re-label (clean-candidate rule) / pull them into the candidate set (once)
            const uint32_t kb = __float_as_uint(fminf(tau, m));
            // The marks of the whole ring are requested first (no store in that loop, so the loads overlap) and only the
            // unmarked, eligible neighbours take the CAS: testing them one by one in the loop that issues the CAS and the stage
            // write makes twelve dependent L2 round trips of the one evaluation per vertex that activates.
            uint32_t todo = 0u;
            if (act_now) {
#pragma unroll
              for (int k = 0; k < (int)ELL_W; ++k) {
                const int4 ix = __ldg(&a.ell_idx[(size_t)c * ELL_W + k]);
                if (ix.x == ELL_EMPTY) continue;
                if (__ldcg(&G.mark[(uint32_t)ix.x]) == MARK_NONE) todo |= 1u << (2 * k);
                if (__ldcg(&G.mark[(uint32_t)ix.y]) == MARK_NONE) todo |= 2u << (2 * k);
              }
            }
            for (int k = 0; k < (int)ELL_W; ++k) {
              const int4 ix = __ldg(&a.ell_idx[(size_t)c * ELL_W + k]);
              if (ix.x == ELL_EMPTY) continue;
              const uint32_t xs[2] = {(uint32_t)ix.x, (uint32_t)ix.y};
#pragma unroll
              for (int t = 0; t < 2; ++t) {
                const uint32_t x = xs[t];
                if (changed) atomicMin(&skw[4 * (size_t)x + buf_now], kb);
                if (((todo >> (2 * k + t)) & 1u) && !(a.invalid && a.invalid[x]) && !((double)__ldg(&a.cost[x]) >= a.cost_limit) &&
                    atomicCAS(&G.mark[x], MARK_NONE, MARK_CAND) == MARK_NONE)
                  batch_stage_write(st, atomicAdd(&st.n, 1u), x, list_n, count_next);
              }
            }
          }
        }
        const unsigned dm = __ballot_sync(FULL, done), fm = __ballot_sync(FULL, has && defer);
        if (dm) {   // the candidate survives into the next round's list (one shared atomic per warp)
          const unsigned int base = warp_reserve(&st.n, (unsigned)__popc(dm));
          if (done) batch_stage_write(st, base + __popc(dm & lt), c | (((ce & LIST_ACTIVATED) || act_now) ? LIST_ACTIVATED : 0u), list_n, count_next);
        }
        if (fm) {
          const unsigned int base = warp_reserve(&wk.ns, (unsigned)__popc(fm));
          if (has && defer) wk.sq[base + __popc(fm & lt)] = ce;
        }
      }
      __syncthreads();
      if (wk.ns) batch_general_phase(a, G, sd, st, wk, list_n, count_next, band_end, strict, r, my_mtau, my_lo, my_recomputes);   // phase C (block-uniform branch)
      __syncthreads();
      if (threadIdx.x == 0) { wk.n = 0; wk.ns = 0; }
      __syncthreads();
    }     // chunks
    stage_reduce(st, my_mtau, my_lo);
    {   // statistics: one atomic per warp and round
      const unsigned int wr = __reduce_add_sync(FULL, my_recomputes), ws = __reduce_add_sync(FULL, my_settled), wk2 = __reduce_add_sync(FULL, my_skipped);
      if (lane == 0) {
        if (wr) atomicAdd(&ctl->recomputes, (unsigned long long)wr);
        if (ws) atomicAdd(&ctl->settled, (unsigned long long)ws);
        if (wk2) atomicAdd(&ctl->skipped, (unsigned long long)wk2);
      }
      my_recomputes = 0; my_settled = 0; my_skipped = 0;
    }
    stage_flush(st, list_n, count_next, &ctl->m_tau[slot], &ctl->lo[slot]);
    band_end_prev = band_end;
    group_sync<CS>();
  }
  band_wave_end<false>(ctl, gtid, r, a.max_rounds, strict);
#ifdef MNB_EMU_ACTIVE
  group_sync<CS>();
  if (gtid == 0 && getenv("MNB_EMU_TRACE")) fprintf(stderr, "[batch plan] rounds %u evaluations: still-inf %llu changed %llu unchanged %llu (general path %llu) settled %llu\n", r, ctl->t_ph[0], ctl->t_ph[1], ctl->t_ph[2], ctl->t_ph[3], ctl->settled);
#endif
}

}  // namespace mnb
