// Inflation repair (mnb_inflation_repair): the delta of the lethal set and the invalid mask, the resident cluster ids of
// the inflation footprint, the affected region, the patch of the resident result and the ordered changed set.  The wave
// itself is k_inflate seeded with the lethals of the affected clusters; DESIGN §4 has the argument why that is exact.
// (part of libmeshnav_b200.so: included by meshnav.cu, which holds the C ABI and all host code)
#pragma once
#include "launch.cuh"
#include "kernels_field.cuh"

using namespace mnb;

// Footprint = the vertices with a finite distances_ entry; a cluster = a connected component of the footprint, two
// footprint vertices linked when they share a face.  Cluster id = the smallest vertex id of the cluster; not in the
// footprint: CLUSTER_NONE.
constexpr uint32_t CLUSTER_NONE = 0xffffffffu;

__device__ __forceinline__ bool ir_bit(const uint32_t* __restrict__ bits, uint32_t v) { return (bits[v >> 5] >> (v & 31u)) & 1u; }
__device__ __forceinline__ void ir_set(uint32_t* bits, uint32_t v) {
  const uint32_t m = 1u << (v & 31u);
  if (!(__ldcg(&bits[v >> 5]) & m)) atomicOr(&bits[v >> 5], m);
}
__device__ __forceinline__ bool ir_finite(float d) { return __float_as_uint(d) != INF_BITS; }

// ---- cluster ids: union-find on the id array itself; a root hooks under the smaller root, so every root is the smallest
// id of its tree.  Concurrent unites are safe: only a root's parent is ever CAS-ed, and path halving stores an ancestor.
__device__ __forceinline__ uint32_t uf_find(uint32_t* P, uint32_t x) {
  for (;;) {
    const uint32_t p = __ldcg(&P[x]);
    if (p == x) return x;
    const uint32_t g = __ldcg(&P[p]);
    if (g != p) P[x] = g;
    x = g;
  }
}
__device__ __forceinline__ void uf_unite(uint32_t* P, uint32_t a, uint32_t b) {
  for (;;) {
    a = uf_find(P, a); b = uf_find(P, b);
    if (a == b) return;
    if (a > b) { const uint32_t t = a; a = b; b = t; }
    if (atomicCAS(&P[b], b, a) == b) return;
  }
}

struct ClusterArgs {
  uint32_t V;
  const uint32_t* cor_ptr; const int4* cor_idx;
  const float* dist;           // resident distances_: finite = footprint
  uint32_t* cid;
  const uint32_t* list; uint32_t n;   // the vertices to work on; null = all V
};
__device__ __forceinline__ bool cluster_vertex(const ClusterArgs& a, uint32_t& x) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (a.list ? a.n : a.V)) return false;
  x = a.list ? a.list[i] : i;
  return true;
}
__global__ void __launch_bounds__(256) k_cluster_init(const ClusterArgs a) {
  uint32_t x;
  if (cluster_vertex(a, x)) a.cid[x] = ir_finite(a.dist[x]) ? x : CLUSTER_NONE;
}
// every face links its footprint vertices: x unites with the smaller-id footprint vertices of each incident face
__global__ void __launch_bounds__(256) k_cluster_unite(const ClusterArgs a) {
  uint32_t x;
  if (!cluster_vertex(a, x) || !ir_finite(a.dist[x])) return;
  for (uint32_t k = a.cor_ptr[x]; k < a.cor_ptr[x + 1]; ++k) {
    const int4 ix = a.cor_idx[k];
    const uint32_t u[2] = {(uint32_t)ix.x, (uint32_t)ix.y};
    for (int t = 0; t < 2; ++t)
      if (u[t] < x && ir_finite(a.dist[u[t]])) uf_unite(a.cid, x, u[t]);
  }
}
// after the unites: every vertex points at its root (read-only walk; other threads only shorten the chains it reads)
__global__ void __launch_bounds__(256) k_cluster_flatten(const ClusterArgs a) {
  uint32_t x;
  if (!cluster_vertex(a, x)) return;
  uint32_t r = a.cid[x];
  if (r == CLUSTER_NONE) return;
  for (uint32_t p = __ldcg(&a.cid[r]); p != r; p = __ldcg(&a.cid[r])) r = p;
  a.cid[x] = r;
}

struct InflRepairArgs {
  uint32_t V;
  const uint32_t* cor_ptr; const int4* cor_idx;
  const uint32_t* cid;                       // cluster ids of the previous result
  const uint32_t* old_bits; const uint32_t* new_bits;   // lethal sets of the previous call and of this one (bitmaps)
  const uint8_t* old_inv; const uint8_t* new_inv;       // invalid masks (null = none invalid)
  uint32_t* aff;                             // affected clusters, bitmap over cluster ids
  const uint32_t* lethals; uint32_t n_lethals;          // the new lethal set as the caller passed it
  uint32_t* seeds;
  unsigned int* cnt;                         // [0] delta vertices, [1] seeds, [2] merge check added a cluster, [3] region size,
                                             // [4] old footprint, [5] its vertices in affected clusters
};

__global__ void __launch_bounds__(256) k_lethal_bits(const uint32_t* __restrict__ lethals, uint32_t n, uint32_t V, uint32_t* bits) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t v = lethals[i];
  if (v < V) ir_set(bits, v);                // ids >= V are ignored, as k_inflate ignores them
}

// delta = lethal-set symmetric difference + invalid-flag flips; its clusters and the clusters sharing a face with it
// are affected
__global__ void __launch_bounds__(256) k_infl_delta(const InflRepairArgs a) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= a.V) return;
  const bool iold = a.old_inv && a.old_inv[v], inew = a.new_inv && a.new_inv[v];
  if (ir_bit(a.old_bits, v) == ir_bit(a.new_bits, v) && iold == inew) return;
  atomicAdd(&a.cnt[0], 1u);
  if (a.cid[v] != CLUSTER_NONE) ir_set(a.aff, a.cid[v]);
  for (uint32_t k = a.cor_ptr[v]; k < a.cor_ptr[v + 1]; ++k) {
    const int4 ix = a.cor_idx[k];
    const uint32_t c1 = a.cid[ix.x], c2 = a.cid[ix.y];
    if (c1 != CLUSTER_NONE) ir_set(a.aff, c1);
    if (c2 != CLUSTER_NONE) ir_set(a.aff, c2);
  }
}

// the size of the old footprint and of its affected part, from which the host chooses the whole-map wave
__global__ void __launch_bounds__(256) k_infl_affected_count(const InflRepairArgs a) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t c = v < a.V ? a.cid[v] : CLUSTER_NONE;
  const unsigned int foot = __reduce_add_sync(0xffffffffu, c != CLUSTER_NONE ? 1u : 0u);
  const unsigned int hit = __reduce_add_sync(0xffffffffu, c != CLUSTER_NONE && ir_bit(a.aff, c) ? 1u : 0u);
  if ((threadIdx.x & 31) == 0) {
    if (foot) atomicAdd(&a.cnt[4], foot);
    if (hit) atomicAdd(&a.cnt[5], hit);
  }
}

// seeds of the local wave: the new lethals in an affected cluster or outside the old footprint
__global__ void __launch_bounds__(256) k_infl_seeds(const InflRepairArgs a) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.n_lethals) return;
  const uint32_t v = a.lethals[i];
  if (v >= a.V) return;
  const uint32_t c = a.cid[v];
  if (c == CLUSTER_NONE || ir_bit(a.aff, c)) a.seeds[atomicAdd(&a.cnt[1], 1u)] = v;
}

// the new footprint N (finite local labels) must not touch an unaffected cluster: a face holding a vertex of N and a
// footprint vertex of an unaffected cluster makes that cluster affected, and the wave runs again
__global__ void __launch_bounds__(256) k_infl_merge_check(const InflRepairArgs a, const float* __restrict__ local_dist) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= a.V || !ir_finite(local_dist[v])) return;
  auto check = [&](uint32_t c) {
    if (c != CLUSTER_NONE && !ir_bit(a.aff, c)) { ir_set(a.aff, c); a.cnt[2] = 1u; }
  };
  check(a.cid[v]);
  for (uint32_t k = a.cor_ptr[v]; k < a.cor_ptr[v + 1]; ++k) {
    const int4 ix = a.cor_idx[k];
    check(a.cid[ix.x]); check(a.cid[ix.y]);
  }
}

// Region = the affected old footprint + N (all = every vertex: the whole-map path).  Inside it the local wave's result
// replaces the resident one (+inf / NaN where the old footprint lost its entry); outside it every bit stays.  out_dist /
// out_cost hold the local wave's dense output on entry (k_inflate wrote them) and the full new result on exit.
struct InflPatchArgs {
  uint32_t V; int all;
  const uint32_t* aff; uint32_t* cid;        // cid: null on the whole-map path (the ids are recomputed lazily)
  float* out_dist; float* out_cost;
  float* res_dist; float* res_risk; int has_risk;   // resident distances_ and riskiness (the previous result)
  uint32_t* chg_bits;                        // riskiness entry changed (presence or value bits; NaN == NaN)
  uint32_t* region; unsigned int* n_region;
};
__global__ void __launch_bounds__(256) k_infl_patch(const InflPatchArgs a) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= a.V) return;
  const float ld = a.out_dist[v];
  const bool in_n = ir_finite(ld);
  bool region = a.all != 0 || in_n;
  if (!region) { const uint32_t c = a.cid[v]; region = c != CLUSTER_NONE && ir_bit(a.aff, c); }
  if (!region) {
    a.out_dist[v] = a.res_dist[v]; a.out_cost[v] = a.res_risk[v];
    return;
  }
  const float r = a.out_cost[v];
  const float old = a.has_risk ? a.res_risk[v] : __int_as_float(0x7fc00000);
  if (__float_as_uint(r) != __float_as_uint(old) && !(r != r && old != old)) atomicOr(&a.chg_bits[v >> 5], 1u << (v & 31u));
  a.res_dist[v] = ld; a.res_risk[v] = r;
  if (a.cid) { a.cid[v] = in_n ? v : CLUSTER_NONE; a.region[atomicAdd(a.n_region, 1u)] = v; }
}

// ordered compaction of a bitmap: per-tile counts, k_update_set_scan over them, ordered write
constexpr int BITS_TILE_WORDS = 256;       // one word per thread
__global__ void __launch_bounds__(256) k_bits_count(const uint32_t* __restrict__ bits, uint32_t n_words, unsigned int* __restrict__ tile_count) {
  __shared__ unsigned int cnt;
  if (threadIdx.x == 0) cnt = 0;
  __syncthreads();
  const uint32_t w = blockIdx.x * (uint32_t)BITS_TILE_WORDS + threadIdx.x;
  const unsigned int wsum = __reduce_add_sync(0xffffffffu, w < n_words ? (unsigned int)__popc(bits[w]) : 0u);
  if ((threadIdx.x & 31) == 0 && wsum) atomicAdd(&cnt, wsum);
  __syncthreads();
  if (threadIdx.x == 0) tile_count[blockIdx.x] = cnt;
}
__global__ void __launch_bounds__(256) k_bits_write(const uint32_t* __restrict__ bits, uint32_t n_words,
                                                    const unsigned int* __restrict__ tile_offset, uint32_t* __restrict__ out) {
  __shared__ unsigned int warp_sum[8];
  const uint32_t w = blockIdx.x * (uint32_t)BITS_TILE_WORDS + threadIdx.x;
  uint32_t word = w < n_words ? bits[w] : 0u;
  const unsigned int x = (unsigned int)__popc(word);
  unsigned int incl = x;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const unsigned int y = __shfl_up_sync(0xffffffffu, incl, o); if ((int)(threadIdx.x & 31) >= o) incl += y; }
  if ((threadIdx.x & 31) == 31) warp_sum[threadIdx.x >> 5] = incl;
  __syncthreads();
  unsigned int pos = tile_offset[blockIdx.x] + incl - x;
  for (uint32_t q = 0; q < (threadIdx.x >> 5); ++q) pos += warp_sum[q];
  while (word) {
    const int b = __ffs(word) - 1;
    out[pos++] = 32u * w + (uint32_t)b;
    word &= word - 1u;
  }
}

// the repulsive field of the region's vertices (k_infl_vec_* over a vertex list)
__global__ void __launch_bounds__(128) k_infl_vec_lethal_list(const InflVecArgs a, const uint32_t* __restrict__ list, uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) infl_vec_lethal_at(a, list[i]);
}
__global__ void __launch_bounds__(128) k_infl_vec_sources_list(const InflVecArgs a, const uint32_t* __restrict__ list, uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) infl_vec_sources_at(a, list[i]);
}
__global__ void __launch_bounds__(256) k_infl_vec_sweep_list(const InflVecArgs a, const uint32_t* __restrict__ list, uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) infl_vec_sweep_at(a, list[i]);
}
