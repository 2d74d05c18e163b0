// Fused geometric cost layers + MaxCombination + lethal masks, face / vertex normals.
// (part of libmeshnav_b200.so: included by meshnav.cu, which holds the C ABI and all host code)
#pragma once
#include "launch.cuh"
#include "../../include/meshnav_b200.h"
#include "band_engine.cuh"

using namespace mnb;

// ============================================================================
// Fused geometric cost layers (mesh_layers: HeightDiff, Roughness, Steepness, Ridge, Clearance cost
// mapping, Border) + MaxCombinationLayer + lethal masks: ONE pass over the radius neighbourhood per
// vertex instead of the reference's three independent visitLocalVertexNeighborhood runs with
// std::set bookkeeping (ridge_layer.cpp:166-175, height_diff_layer.cpp:108, roughness_layer.cpp:143).
// Definitions of the lvr2 pieces: see oracle/oracle.cpp (orc_layers).
// ============================================================================
__global__ void k_face_normals(const float* __restrict__ pos, const uint32_t* __restrict__ faces, uint32_t F,
                               float* __restrict__ fn) {
  const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const float* p0 = pos + 3 * (size_t)faces[3 * (size_t)f];
  const float* p1 = pos + 3 * (size_t)faces[3 * (size_t)f + 1];
  const float* p2 = pos + 3 * (size_t)faces[3 * (size_t)f + 2];
  const float ax = p1[0] - p0[0], ay = p1[1] - p0[1], az = p1[2] - p0[2];
  const float bx = p2[0] - p0[0], by = p2[1] - p0[1], bz = p2[2] - p0[2];
  float nx = ay * bz - az * by, ny = az * bx - ax * bz, nz = ax * by - ay * bx;
  const float l = sqrtf(nx * nx + ny * ny + nz * nz);
  if (l > 0) { nx /= l; ny /= l; nz /= l; }
  fn[3 * (size_t)f] = nx; fn[3 * (size_t)f + 1] = ny; fn[3 * (size_t)f + 2] = nz;
}

__global__ void k_vertex_normals(const uint32_t* __restrict__ cor_ptr, const int4* __restrict__ cor_idx,
                                 const float* __restrict__ fn, uint32_t V, float* __restrict__ vn) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  float nx = 0, ny = 0, nz = 0;
  for (uint32_t k = cor_ptr[v]; k < cor_ptr[v + 1]; ++k) {
    const int f = cor_idx[k].z;
    nx = nx + fn[3 * (size_t)f]; ny = ny + fn[3 * (size_t)f + 1]; nz = nz + fn[3 * (size_t)f + 2];
  }
  const float l = sqrtf(nx * nx + ny * ny + nz * nz);
  if (l > 0) { nx /= l; ny /= l; nz /= l; }
  vn[3 * (size_t)v] = nx; vn[3 * (size_t)v + 1] = ny; vn[3 * (size_t)v + 2] = nz;
}

// acos of a float as the layers use it (roughness: angle between normals, steepness_layer.cpp:165): evaluated in double and
// rounded once.  The reference calls the float overload of its libm, whose last bit differs between libm versions and
// from CUDA's acosf; lethal sets are threshold tests on these values, so both this kernel and the oracle use the value
// that is well defined everywhere -- the correctly rounded one (double acos is accurate to < 2 ulp of double on both sides).
__device__ __forceinline__ float acos_f(float x) { return (float)acos((double)x); }

struct LayerKernelArgs {
  uint32_t V;
  const float* pos; const float* vn;
  const uint32_t* adj_ptr; const uint32_t* adj_nbr;
  const uint8_t* border;
  const float* clearance;      // may be null
  mnb_layer_params P;
  float* costs;                // 6 x V
  float* combined; uint8_t* lethal_mask;
  unsigned int* overflow;      // neighbourhood larger than the per-thread scratch
  // packed copies for k_layers<true>: one 16-byte load per position / normal, one 32-byte row of neighbour ids per vertex
  const float4* pos4; const float4* vn4; const uint4* nbr8;
};

// k_layers<true> reads packed copies of the same data: every per-thread (scattered) load instruction costs 32 L1
// wavefronts whatever its width, so {x,y,z} as three 4-byte loads and a neighbour list behind two CSR pointers triple the
// wavefront count of the walk, which is what bounds the kernel (DESIGN.md 5).
constexpr uint32_t NBR8_EMPTY = 0xffffffffu, NBR8_BIG = 0xfffffffeu;
__global__ void k_pack_layers(const float* __restrict__ pos, const float* __restrict__ vn, const uint32_t* __restrict__ adj_ptr,
                              const uint32_t* __restrict__ adj_nbr, uint32_t V, float4* __restrict__ pos4, float4* __restrict__ vn4,
                              uint32_t* __restrict__ nbr8) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  pos4[v] = make_float4(pos[3 * (size_t)v], pos[3 * (size_t)v + 1], pos[3 * (size_t)v + 2], 0.0f);
  vn4[v] = make_float4(vn[3 * (size_t)v], vn[3 * (size_t)v + 1], vn[3 * (size_t)v + 2], 0.0f);
  const uint32_t kb = adj_ptr[v], deg = adj_ptr[v + 1] - kb;
  for (uint32_t j = 0; j < 8; ++j)      // CSR order (ascending edge id) is kept: the traversal order must not change
    nbr8[8 * (size_t)v + j] = deg > 8 ? NBR8_BIG : (j < deg ? adj_nbr[kb + j] : NBR8_EMPTY);
}

constexpr int NB_SEEN = 320, NB_STACK = 160;

// (fallback for neighbourhoods that overflow the hashed set below: linear `seen` list, any size up to NB_SEEN)
// traversal shared by the three radius layers; WHICH selects the accumulators that are active (bit0 height
// diff, bit1 roughness, bit2 ridge) so that layers with equal radii share one walk
template <int WHICH>
__device__ __noinline__ void walk_linear(const LayerKernelArgs& a, uint32_t v, float radius, float& zmin, float& zmax,
                                     float& rsum, int& rcnt, float& value, int& num) {
  uint32_t seen[NB_SEEN]; uint32_t stack[NB_STACK];
  int ns = 0, sp = 0;
  seen[ns++] = v; stack[sp++] = v;
  const float px = a.pos[3 * (size_t)v], py = a.pos[3 * (size_t)v + 1], pz = a.pos[3 * (size_t)v + 2];
  const float nvx = a.vn[3 * (size_t)v], nvy = a.vn[3 * (size_t)v + 1], nvz = a.vn[3 * (size_t)v + 2];
  const float rx = px + nvx, ry = py + nvy, rz = pz + nvz;
  while (sp > 0) {
    const uint32_t u = stack[--sp];
    for (uint32_t k = a.adj_ptr[u]; k < a.adj_ptr[u + 1]; ++k) {
      const uint32_t n = a.adj_nbr[k];
      bool was = false;
      for (int s = 0; s < ns; ++s) if (seen[s] == n) { was = true; break; }
      if (was) continue;
      if (ns >= NB_SEEN) { atomicAdd(a.overflow, 1u); return; }
      seen[ns++] = n;
      const float qx = a.pos[3 * (size_t)n], qy = a.pos[3 * (size_t)n + 1], qz = a.pos[3 * (size_t)n + 2];
      const float dx = qx - px, dy = qy - py, dz = qz - pz;
      if (sqrtf(dx * dx + dy * dy + dz * dz) < radius) {
        if (WHICH & 1) { zmin = fminf(zmin, qz); zmax = fmaxf(zmax, qz); }
        if (WHICH & 6) {
          const float nnx = a.vn[3 * (size_t)n], nny = a.vn[3 * (size_t)n + 1], nnz = a.vn[3 * (size_t)n + 2];
          if (WHICH & 2) {
            float dot = nvx * nnx + nvy * nny + nvz * nnz;
            dot = fminf(1.0f, fmaxf(-1.0f, dot));
            rsum = rsum + acos_f(dot); rcnt++;
          }
          if (WHICH & 4) {
            const float cx = (qx + nnx) - rx, cy = (qy + nny) - ry, cz = (qz + nnz) - rz;
            value += sqrtf(cx * cx + cy * cy + cz * cz); num++;
          }
        }
        if (sp >= NB_STACK) { atomicAdd(a.overflow, 1u); return; }
        stack[sp++] = n;
      }
    }
  }
}


// Same traversal, same visiting order (so the float sums are bit-identical to the oracle's), but the `seen` set is a
// 128-entry open-addressing hash in local memory instead of a linear list: ~2 probes per membership test instead of
// ~24 compares.  Neighbourhoods with more than NB_HSEEN seen vertices fall back to walk_linear.
constexpr int NB_HASH = 128, NB_HSEEN = 96;
template <int WHICH>
__device__ __forceinline__ void walk(const LayerKernelArgs& a, uint32_t v, float radius, float& zmin, float& zmax,
                                     float& rsum, int& rcnt, float& value, int& num) {
  uint32_t ht[NB_HASH]; uint32_t stack[NB_HSEEN];
#pragma unroll 8
  for (int i = 0; i < NB_HASH; ++i) ht[i] = 0xffffffffu;
  const float zmin0 = zmin, zmax0 = zmax, rsum0 = rsum, value0 = value; const int rcnt0 = rcnt, num0 = num;
  int ns = 0, sp = 0;
  ht[(v * 2654435761u) >> 25] = v; ns = 1; stack[sp++] = v;
  const float px = a.pos[3 * (size_t)v], py = a.pos[3 * (size_t)v + 1], pz = a.pos[3 * (size_t)v + 2];
  const float nvx = a.vn[3 * (size_t)v], nvy = a.vn[3 * (size_t)v + 1], nvz = a.vn[3 * (size_t)v + 2];
  const float rx = px + nvx, ry = py + nvy, rz = pz + nvz;
  bool overflow = false;
  while (sp > 0 && !overflow) {
    const uint32_t u = stack[--sp];
    for (uint32_t k = a.adj_ptr[u]; k < a.adj_ptr[u + 1]; ++k) {
      const uint32_t n = a.adj_nbr[k];
      uint32_t h = (n * 2654435761u) >> 25;
      bool was = false;
      for (;;) {
        const uint32_t e = ht[h];
        if (e == n) { was = true; break; }
        if (e == 0xffffffffu) break;
        h = (h + 1u) & (uint32_t)(NB_HASH - 1);
      }
      if (was) continue;
      if (ns >= NB_HSEEN) { overflow = true; break; }
      ht[h] = n; ++ns;
      const float qx = a.pos[3 * (size_t)n], qy = a.pos[3 * (size_t)n + 1], qz = a.pos[3 * (size_t)n + 2];
      const float dx = qx - px, dy = qy - py, dz = qz - pz;
      if (sqrtf(dx * dx + dy * dy + dz * dz) < radius) {
        if (WHICH & 1) { zmin = fminf(zmin, qz); zmax = fmaxf(zmax, qz); }
        if (WHICH & 6) {
          const float nnx = a.vn[3 * (size_t)n], nny = a.vn[3 * (size_t)n + 1], nnz = a.vn[3 * (size_t)n + 2];
          if (WHICH & 2) {
            float dot = nvx * nnx + nvy * nny + nvz * nnz;
            dot = fminf(1.0f, fmaxf(-1.0f, dot));
            rsum = rsum + acos_f(dot); rcnt++;
          }
          if (WHICH & 4) {
            const float cx = (qx + nnx) - rx, cy = (qy + nny) - ry, cz = (qz + nnz) - rz;
            value += sqrtf(cx * cx + cy * cy + cz * cz); num++;
          }
        }
        stack[sp++] = n;            // sp <= ns <= NB_HSEEN
      }
    }
  }
  if (overflow) {
    zmin = zmin0; zmax = zmax0; rsum = rsum0; value = value0; rcnt = rcnt0; num = num0;
    walk_linear<WHICH>(a, v, radius, zmin, zmax, rsum, rcnt, value, num);
  }
}

// Variant with the `seen` hash set and the traversal stack in SHARED memory (slot-major, one bank per thread: conflict
// free) instead of thread-local memory: 1536 resident threads x ~0.9 KB of randomly probed local memory does not fit the
// L1, so every probe of the local-memory version is an L2 trip.  Same traversal, same visiting order, same sums.
// Opt-in (MNB_LAYERS_SMEM=1).
constexpr int LS_THREADS = 128, LS_STACK = 48;
template <int WHICH>
__device__ __forceinline__ void walk_smem(const LayerKernelArgs& a, uint32_t v, float radius, float& zmin, float& zmax,
                                          float& rsum, int& rcnt, float& value, int& num, uint32_t* __restrict__ ht,
                                          uint32_t* __restrict__ stack) {
  // ht[slot * LS_THREADS], stack[i * LS_THREADS]: both already offset by threadIdx.x
#pragma unroll 8
  for (int i = 0; i < NB_HASH; ++i) ht[i * LS_THREADS] = 0xffffffffu;
  const float zmin0 = zmin, zmax0 = zmax, rsum0 = rsum, value0 = value; const int rcnt0 = rcnt, num0 = num;
  int ns = 0, sp = 0;
  ht[((v * 2654435761u) >> 25) * LS_THREADS] = v; ns = 1; stack[(sp++) * LS_THREADS] = v;
  const float4 pv = __ldg(&a.pos4[v]), nv = __ldg(&a.vn4[v]);
  const float px = pv.x, py = pv.y, pz = pv.z;
  const float nvx = nv.x, nvy = nv.y, nvz = nv.z;
  const float rx = px + nvx, ry = py + nvy, rz = pz + nvz;
  bool overflow = false;
  // one neighbour of the vertex being expanded: same body as walk<>, on the packed arrays
  auto visit = [&](uint32_t n) {
    uint32_t h = (n * 2654435761u) >> 25;
    for (;;) {
      const uint32_t e = ht[h * LS_THREADS];
      if (e == n) return;
      if (e == 0xffffffffu) break;
      h = (h + 1u) & (uint32_t)(NB_HASH - 1);
    }
    if (ns >= NB_HSEEN) { overflow = true; return; }
    ht[h * LS_THREADS] = n; ++ns;
    const float4 q = __ldg(&a.pos4[n]);
    const float qx = q.x, qy = q.y, qz = q.z;
    const float dx = qx - px, dy = qy - py, dz = qz - pz;
    if (sqrtf(dx * dx + dy * dy + dz * dz) < radius) {
      if (WHICH & 1) { zmin = fminf(zmin, qz); zmax = fmaxf(zmax, qz); }
      if (WHICH & 6) {
        const float4 nn = __ldg(&a.vn4[n]);
        const float nnx = nn.x, nny = nn.y, nnz = nn.z;
        if (WHICH & 2) {
          float dot = nvx * nnx + nvy * nny + nvz * nnz;
          dot = fminf(1.0f, fmaxf(-1.0f, dot));
          rsum = rsum + acos_f(dot); rcnt++;
        }
        if (WHICH & 4) {
          const float cx = (qx + nnx) - rx, cy = (qy + nny) - ry, cz = (qz + nnz) - rz;
          value += sqrtf(cx * cx + cy * cy + cz * cz); num++;
        }
      }
      if (sp >= LS_STACK) { overflow = true; return; }
      stack[(sp++) * LS_THREADS] = n;
    }
  };
  while (sp > 0 && !overflow) {
    const uint32_t u = stack[(--sp) * LS_THREADS];
    const uint4 r0 = __ldg(&a.nbr8[2 * (size_t)u]);
    if (r0.x == NBR8_BIG) {                       // more than 8 neighbours: CSR row
      for (uint32_t k = a.adj_ptr[u]; k < a.adj_ptr[u + 1] && !overflow; ++k) visit(a.adj_nbr[k]);
      continue;
    }
    const uint4 r1 = __ldg(&a.nbr8[2 * (size_t)u + 1]);
    const uint32_t ids[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (ids[j] == NBR8_EMPTY || overflow) break;
      visit(ids[j]);
    }
  }
  if (overflow) {
    zmin = zmin0; zmax = zmax0; rsum = rsum0; value = value0; rcnt = rcnt0; num = num0;
    walk_linear<WHICH>(a, v, radius, zmin, zmax, rsum, rcnt, value, num);
  }
}

// Third form of the same traversal (same visiting order, same sums): memory-level parallelism instead of occupancy.  The
// walk is a chain of dependent loads -- pop u, load u's neighbour row, then per neighbour: hash probe -> position ->
// (inside the radius) normal -- ~13 L2 round trips per expanded vertex, which is what the 9.6 ms of the per-thread forms
// are made of (round 2 ncu: 18 % issue utilisation, everything on the long scoreboard; the shared-memory hash alone
// changed nothing).  Here the positions AND normals of all (up to 8) neighbours of u are requested up front, 16 independent
// 16-byte loads in flight per thread, before the first hash probe; the sequential part then runs on registers.  Seen-set and
// stack live in shared memory (slot-major: conflict free) with T threads per CTA.
template <int WHICH, int T>
__device__ __forceinline__ void walk_pf(const LayerKernelArgs& a, uint32_t v, float radius, float& zmin, float& zmax,
                                        float& rsum, int& rcnt, float& value, int& num, uint32_t* __restrict__ ht,
                                        uint32_t* __restrict__ stack) {
#pragma unroll 8
  for (int i = 0; i < NB_HASH; ++i) ht[i * T] = 0xffffffffu;
  const float zmin0 = zmin, zmax0 = zmax, rsum0 = rsum, value0 = value; const int rcnt0 = rcnt, num0 = num;
  int ns = 0, sp = 0;
  ht[((v * 2654435761u) >> 25) * T] = v; ns = 1; stack[(sp++) * T] = v;
  const float4 pv = __ldg(&a.pos4[v]), nv = __ldg(&a.vn4[v]);
  const float px = pv.x, py = pv.y, pz = pv.z;
  const float nvx = nv.x, nvy = nv.y, nvz = nv.z;
  const float rx = px + nvx, ry = py + nvy, rz = pz + nvz;
  bool overflow = false;
  auto visit = [&](uint32_t n, const float4& q, const float4& nn) {
    uint32_t h = (n * 2654435761u) >> 25;
    for (;;) {
      const uint32_t e = ht[h * T];
      if (e == n) return;
      if (e == 0xffffffffu) break;
      h = (h + 1u) & (uint32_t)(NB_HASH - 1);
    }
    if (ns >= NB_HSEEN) { overflow = true; return; }
    ht[h * T] = n; ++ns;
    const float qx = q.x, qy = q.y, qz = q.z;
    const float dx = qx - px, dy = qy - py, dz = qz - pz;
    if (sqrtf(dx * dx + dy * dy + dz * dz) < radius) {
      if (WHICH & 1) { zmin = fminf(zmin, qz); zmax = fmaxf(zmax, qz); }
      if (WHICH & 6) {
        const float nnx = nn.x, nny = nn.y, nnz = nn.z;
        if (WHICH & 2) {
          float dot = nvx * nnx + nvy * nny + nvz * nnz;
          dot = fminf(1.0f, fmaxf(-1.0f, dot));
          rsum = rsum + acos_f(dot); rcnt++;
        }
        if (WHICH & 4) {
          const float cx = (qx + nnx) - rx, cy = (qy + nny) - ry, cz = (qz + nnz) - rz;
          value += sqrtf(cx * cx + cy * cy + cz * cz); num++;
        }
      }
      if (sp >= LS_STACK) { overflow = true; return; }
      stack[(sp++) * T] = n;
      mnb_prefetch_l2(a.nbr8 + 2 * (size_t)n);   // its row is needed when it is popped
    }
  };
  while (sp > 0 && !overflow) {
    const uint32_t u = stack[(--sp) * T];
    const uint4 r0 = __ldg(&a.nbr8[2 * (size_t)u]);
    if (r0.x == NBR8_BIG) {                       // more than 8 neighbours: CSR row, one at a time
      for (uint32_t k = a.adj_ptr[u]; k < a.adj_ptr[u + 1] && !overflow; ++k) { const uint32_t n = a.adj_nbr[k]; visit(n, __ldg(&a.pos4[n]), __ldg(&a.vn4[n])); }
      continue;
    }
    const uint4 r1 = __ldg(&a.nbr8[2 * (size_t)u + 1]);
    const uint32_t ids[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
    float4 q[8], nn[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {                 // all requests first ...
      const uint32_t n = ids[j] == NBR8_EMPTY ? v : ids[j];
      q[j] = __ldg(&a.pos4[n]);
      if (WHICH & 6) nn[j] = __ldg(&a.vn4[n]);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {                 // ... then the sequential part, in the reference's order
      if (ids[j] == NBR8_EMPTY || overflow) break;
      visit(ids[j], q[j], nn[j]);
    }
  }
  if (overflow) {
    zmin = zmin0; zmax = zmax0; rsum = rsum0; value = value0; rcnt = rcnt0; num = num0;
    walk_linear<WHICH>(a, v, radius, zmin, zmax, rsum, rcnt, value, num);
  }
}

// Fourth form: walk_pf with a COMPACT seen-set.  The 704 bytes of shared memory a thread of walk_pf owns (128 x 4-byte hash
// entries + 48 x 4-byte stack) cap the kernel at 10 resident warps per SM, and it is bound by instruction issue at that
// occupancy (ncu: 34 % issue utilisation at 15 % active warps).  Vertex ids inside one neighbourhood are close to the centre's
// id on any mesh whose numbering has spatial locality (scan order, Morton order, most reconstruction outputs), so the hash
// stores 16-bit codes  n - v + 32768  (0 = empty) and the stack the 8-bit hash slot of the vertex: 304 bytes per thread, 18
// resident warps.  A neighbour whose id is further than 32767 from the centre's raises `overflow` like a full table does:
// the vertex is redone by walk_linear -- same traversal order, same sums, so every output stays bit-identical.
template <int WHICH, int T>
__device__ __forceinline__ void walk_pf16(const LayerKernelArgs& a, uint32_t v, float radius, float& zmin, float& zmax,
                                          float& rsum, int& rcnt, float& value, int& num, uint16_t* __restrict__ ht,
                                          uint8_t* __restrict__ stack) {
#pragma unroll 8
  for (int i = 0; i < NB_HASH; ++i) ht[i * T] = 0;
  const float zmin0 = zmin, zmax0 = zmax, rsum0 = rsum, value0 = value; const int rcnt0 = rcnt, num0 = num;
  int ns = 0, sp = 0;
  { const uint32_t h0 = (v * 2654435761u) >> 25; ht[h0 * T] = (uint16_t)32768u; ns = 1; stack[(sp++) * T] = (uint8_t)h0; }
  const float4 pv = __ldg(&a.pos4[v]), nv = __ldg(&a.vn4[v]);
  const float px = pv.x, py = pv.y, pz = pv.z;
  const float nvx = nv.x, nvy = nv.y, nvz = nv.z;
  const float rx = px + nvx, ry = py + nvy, rz = pz + nvz;
  bool overflow = false;
  auto visit = [&](uint32_t n, const float4& q, const float4& nn) {
    const uint32_t code32 = n - v + 32768u;                       // wraps for n < v; in range <=> 1 <= code32 <= 65535
    if (code32 - 1u >= 65535u) { overflow = true; return; }
    const uint16_t code = (uint16_t)code32;
    uint32_t h = (n * 2654435761u) >> 25;
    for (;;) {
      const uint16_t e = ht[h * T];
      if (e == code) return;
      if (e == 0) break;
      h = (h + 1u) & (uint32_t)(NB_HASH - 1);
    }
    if (ns >= NB_HSEEN) { overflow = true; return; }
    ht[h * T] = code; ++ns;
    const float qx = q.x, qy = q.y, qz = q.z;
    const float dx = qx - px, dy = qy - py, dz = qz - pz;
    if (sqrtf(dx * dx + dy * dy + dz * dz) < radius) {
      if (WHICH & 1) { zmin = fminf(zmin, qz); zmax = fmaxf(zmax, qz); }
      if (WHICH & 6) {
        const float nnx = nn.x, nny = nn.y, nnz = nn.z;
        if (WHICH & 2) {
          float dot = nvx * nnx + nvy * nny + nvz * nnz;
          dot = fminf(1.0f, fmaxf(-1.0f, dot));
          rsum = rsum + acos_f(dot); rcnt++;
        }
        if (WHICH & 4) {
          const float cx = (qx + nnx) - rx, cy = (qy + nny) - ry, cz = (qz + nnz) - rz;
          value += sqrtf(cx * cx + cy * cy + cz * cz); num++;
        }
      }
      if (sp >= LS_STACK) { overflow = true; return; }
      stack[(sp++) * T] = (uint8_t)h;
      mnb_prefetch_l2(a.nbr8 + 2 * (size_t)n);   // its row is needed when it is popped
    }
  };
  while (sp > 0 && !overflow) {
    const uint32_t u = v + (uint32_t)ht[(uint32_t)stack[(--sp) * T] * T] - 32768u;
    const uint4 r0 = __ldg(&a.nbr8[2 * (size_t)u]);
    if (r0.x == NBR8_BIG) {                       // more than 8 neighbours: CSR row, one at a time
      for (uint32_t k = a.adj_ptr[u]; k < a.adj_ptr[u + 1] && !overflow; ++k) { const uint32_t n = a.adj_nbr[k]; visit(n, __ldg(&a.pos4[n]), __ldg(&a.vn4[n])); }
      continue;
    }
    const uint4 r1 = __ldg(&a.nbr8[2 * (size_t)u + 1]);
    const uint32_t ids[8] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
    float4 q[8], nn[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {                 // all requests first ...
      const uint32_t n = ids[j] == NBR8_EMPTY ? v : ids[j];
      q[j] = __ldg(&a.pos4[n]);
      if (WHICH & 6) nn[j] = __ldg(&a.vn4[n]);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {                 // ... then the sequential part, in the reference's order
      if (ids[j] == NBR8_EMPTY || overflow) break;
      visit(ids[j], q[j], nn[j]);
    }
  }
  if (overflow) {
    zmin = zmin0; zmax = zmax0; rsum = rsum0; value = value0; rcnt = rcnt0; num = num0;
    walk_linear<WHICH>(a, v, radius, zmin, zmax, rsum, rcnt, value, num);
  }
}

// per-vertex layer values from the accumulators of the walks, lethal bits, MaxCombination
__device__ __forceinline__ void layers_epilogue(const LayerKernelArgs& a, uint32_t v, float zmin, float zmax, float rsum, int rcnt, float value, int num) {
  const mnb_layer_params& P = a.P;
  const float hd = zmax - zmin;
  const float ro = rcnt ? rsum / (float)rcnt : 0.0f;
  const float st = acos_f(a.vn[3 * (size_t)v + 2]);                               // steepness_layer.cpp:165
  const float ri = num == 0 ? (float)(P.ridge_threshold + 0.1) : value / num;     // ridge_layer.cpp:177-184
  const float cl = a.clearance ? a.clearance[v] : __uint_as_float(INF_BITS);
  float cc; bool cl_lethal = false;                                              // clearance_layer.cpp:77-96
  const double inflated_height = P.clearance_robot_height + P.clearance_height_inflation;
  if (cl < P.clearance_robot_height) { cc = 1.0f; cl_lethal = true; }
  else if (cl < inflated_height) {
    const double diff = (cl - P.clearance_robot_height) / P.clearance_height_inflation;
    cc = (float)((cos(diff * 3.14159265358979323846) + 1.0) / 2.0);
  } else cc = 0.0f;
  const float bo = a.border[v] ? (float)P.border_cost : 0.0f;
  const size_t V = a.V;
  if (a.costs) {
    a.costs[v] = hd; a.costs[V + v] = ro; a.costs[2 * V + v] = st; a.costs[3 * V + v] = ri; a.costs[4 * V + v] = cc; a.costs[5 * V + v] = bo;
  }
  uint8_t mask = 0;
  if (hd > P.height_diff_threshold) mask |= 1;
  if (ro > P.roughness_threshold) mask |= 2;
  if (st > P.steepness_threshold) mask |= 4;
  if (ri > P.ridge_threshold) mask |= 8;
  if (cl_lethal) mask |= 16;
  if (bo > P.border_threshold) mask |= 32;
  if (a.lethal_mask) a.lethal_mask[v] = mask;
  if (a.combined) a.combined[v] = fmaxf(fmaxf(fmaxf(0.0f, hd), fmaxf(ro, st)), fmaxf(fmaxf(ri, cc), bo));   // combination_layer.cpp:60-71
}

template <bool SMEM>
__global__ void __launch_bounds__(128) k_layers(const LayerKernelArgs a) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= a.V) return;
  const mnb_layer_params& P = a.P;
  const float pz = a.pos[3 * (size_t)v + 2];
  float zmin = pz, zmax = pz, rsum = 0.0f, value = 0.0f; int rcnt = 0, num = 0;
  const float r_hd = (float)P.height_diff_radius, r_ro = (float)P.roughness_radius, r_ri = (float)P.ridge_radius;
  if constexpr (SMEM) {
    MNB_DYNAMIC_SMEM(ls_raw);
    uint32_t* ht = reinterpret_cast<uint32_t*>(ls_raw) + threadIdx.x;
    uint32_t* stack = ht + NB_HASH * LS_THREADS;
    if (r_hd == r_ro && r_ro == r_ri) {
      walk_smem<7>(a, v, r_hd, zmin, zmax, rsum, rcnt, value, num, ht, stack);
    } else {
      walk_smem<1>(a, v, r_hd, zmin, zmax, rsum, rcnt, value, num, ht, stack);
      walk_smem<2>(a, v, r_ro, zmin, zmax, rsum, rcnt, value, num, ht, stack);
      walk_smem<4>(a, v, r_ri, zmin, zmax, rsum, rcnt, value, num, ht, stack);
    }
  } else if (r_hd == r_ro && r_ro == r_ri) {
    walk<7>(a, v, r_hd, zmin, zmax, rsum, rcnt, value, num);
  } else {
    walk<1>(a, v, r_hd, zmin, zmax, rsum, rcnt, value, num);
    walk<2>(a, v, r_ro, zmin, zmax, rsum, rcnt, value, num);
    walk<4>(a, v, r_ri, zmin, zmax, rsum, rcnt, value, num);
  }
  layers_epilogue(a, v, zmin, zmax, rsum, rcnt, value, num);
}

// the prefetching form (walk_pf) with T threads per CTA; dynamic shared memory = (NB_HASH + LS_STACK) * 4 * T bytes
template <int T>
__global__ void __launch_bounds__(T) k_layers_pf(const LayerKernelArgs a) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= a.V) return;
  const mnb_layer_params& P = a.P;
  const float pz = a.pos[3 * (size_t)v + 2];
  float zmin = pz, zmax = pz, rsum = 0.0f, value = 0.0f; int rcnt = 0, num = 0;
  const float r_hd = (float)P.height_diff_radius, r_ro = (float)P.roughness_radius, r_ri = (float)P.ridge_radius;
  MNB_DYNAMIC_SMEM(ls_raw);
  uint32_t* ht = reinterpret_cast<uint32_t*>(ls_raw) + threadIdx.x;
  uint32_t* stack = ht + NB_HASH * T;
  if (r_hd == r_ro && r_ro == r_ri) {
    walk_pf<7, T>(a, v, r_hd, zmin, zmax, rsum, rcnt, value, num, ht, stack);
  } else {
    walk_pf<1, T>(a, v, r_hd, zmin, zmax, rsum, rcnt, value, num, ht, stack);
    walk_pf<2, T>(a, v, r_ro, zmin, zmax, rsum, rcnt, value, num, ht, stack);
    walk_pf<4, T>(a, v, r_ri, zmin, zmax, rsum, rcnt, value, num, ht, stack);
  }
  layers_epilogue(a, v, zmin, zmax, rsum, rcnt, value, num);
}

// walk_pf16 with T threads per CTA; dynamic shared memory = (2 * NB_HASH + LS_STACK) * T bytes
template <int T, int MINB = 1>
__global__ void __launch_bounds__(T, MINB) k_layers_pf16(const LayerKernelArgs a) {
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= a.V) return;
  const mnb_layer_params& P = a.P;
  const float pz = a.pos[3 * (size_t)v + 2];
  float zmin = pz, zmax = pz, rsum = 0.0f, value = 0.0f; int rcnt = 0, num = 0;
  const float r_hd = (float)P.height_diff_radius, r_ro = (float)P.roughness_radius, r_ri = (float)P.ridge_radius;
  MNB_DYNAMIC_SMEM(ls_raw);
  uint16_t* ht = reinterpret_cast<uint16_t*>(ls_raw) + threadIdx.x;
  uint8_t* stack = reinterpret_cast<uint8_t*>(ls_raw) + 2 * NB_HASH * T + threadIdx.x;
  if (r_hd == r_ro && r_ro == r_ri) {
    walk_pf16<7, T>(a, v, r_hd, zmin, zmax, rsum, rcnt, value, num, ht, stack);
  } else {
    walk_pf16<1, T>(a, v, r_hd, zmin, zmax, rsum, rcnt, value, num, ht, stack);
    walk_pf16<2, T>(a, v, r_ro, zmin, zmax, rsum, rcnt, value, num, ht, stack);
    walk_pf16<4, T>(a, v, r_ri, zmin, zmax, rsum, rcnt, value, num, ht, stack);
  }
  layers_epilogue(a, v, zmin, zmax, rsum, rcnt, value, num);
}
