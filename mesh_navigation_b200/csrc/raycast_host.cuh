// Host side of the ray caster (kernels_raycast.cuh): BVH build on first use, mnb_cast_rays, mnb_obstacle_update /
// mnb_obstacle_reset, mnb_normal_clearance.  Included at the end of meshnav.cu (uses mnb_ctx and its RayCasterState, CK,
// DeviceBuffer, CallerArrays, simple_stats, the ordered compaction kernels of kernels_updates.cuh).
#pragma once
#ifndef MNB_EMU_ACTIVE
#include <cub/device/device_radix_sort.cuh>
#endif

// the kernels' view of the tree: a plain struct of raw pointers, passed by value.  The Morton keys exist during the build only.
static RayBvh ray_bvh(const mnb_ctx* ctx, unsigned long long* keys = nullptr) {
  RayBvh t{};
  t.n = ctx->F; t.eps = ctx->bvh_eps; t.lo = ctx->bvh_lo; t.hi = ctx->bvh_hi; t.parent = ctx->bvh_parent; t.visits = ctx->bvh_visits;
  t.keys = keys; t.order = ctx->bvh_order; t.scene = ctx->bvh_scene;
  return t;
}

// Morton order of the faces: radix sort of (key, face id) pairs on the device (stable: equal keys keep ascending face ids).
// The sorted pairs end up in keys / order.
static int32_t sort_morton(mnb_ctx* ctx, uint32_t n, DeviceBuffer<unsigned long long>& keys, DeviceBuffer<unsigned long long>& keys_tmp,
                           DeviceBuffer<uint32_t>& order, DeviceBuffer<uint32_t>& order_tmp) {
#ifdef MNB_EMU_ACTIVE
  std::vector<uint32_t> idx(n);
  for (uint32_t i = 0; i < n; ++i) idx[i] = i;
  std::stable_sort(idx.begin(), idx.end(), [&](uint32_t a, uint32_t b) { return keys[a] < keys[b]; });
  for (uint32_t i = 0; i < n; ++i) { keys_tmp[i] = keys[idx[i]]; order_tmp[i] = order[idx[i]]; }
#else
  size_t bytes = 0;
  CK(cub::DeviceRadixSort::SortPairs(nullptr, bytes, keys.p, keys_tmp.p, order.p, order_tmp.p, (int)n, 0, 63, ctx->stream));
  DeviceBuffer<unsigned char> tmp;
  CK(tmp.reserve(bytes ? bytes : 1));
  CK(cub::DeviceRadixSort::SortPairs(tmp.p, bytes, keys.p, keys_tmp.p, order.p, order_tmp.p, (int)n, 0, 63, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
#endif
  std::swap(keys, keys_tmp); std::swap(order, order_tmp);
  return MNB_OK;
}

static int32_t build_raycaster(mnb_ctx* ctx) {
  const uint32_t n = ctx->F;
  const size_t nodes = 2 * (size_t)n - 1;
  DeviceBuffer<unsigned long long> keys, keys_tmp; DeviceBuffer<uint32_t> order_tmp;      // of the build: only the tree and the face order are kept
  CK(ctx->bvh_lo.reserve(nodes)); CK(ctx->bvh_hi.reserve(nodes)); CK(ctx->bvh_parent.reserve(nodes)); CK(ctx->bvh_visits.reserve(n));
  CK(keys.reserve(n)); CK(ctx->bvh_order.reserve(n)); CK(keys_tmp.reserve(n)); CK(order_tmp.reserve(n));
  CK(ctx->bvh_scene.reserve(8));
  const unsigned int scene0[8] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u, 0u, 0u};
  CK(cudaMemcpyAsync(ctx->bvh_scene, scene0, sizeof(scene0), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemsetAsync(ctx->bvh_visits, 0, sizeof(unsigned int) * (size_t)n, ctx->stream));
  CK(cudaMemsetAsync(ctx->bvh_parent, 0xff, sizeof(uint32_t) * nodes, ctx->stream));
  MNB_LAUNCH(k_bvh_scene, 2 * ctx->sm_count, 256, 0, ctx->stream, (const float*)ctx->d_pos, ctx->V, ctx->bvh_scene);
  MNB_LAUNCH(k_bvh_morton, (n + 255) / 256, 256, 0, ctx->stream, (const float*)ctx->d_pos, (const uint32_t*)ctx->d_faces, n,
             (const unsigned int*)ctx->bvh_scene, keys, ctx->bvh_order);
  CK(cudaGetLastError());
  unsigned int scene[8];
  CK(cudaMemcpyAsync(scene, ctx->bvh_scene, sizeof(scene), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  float mx; std::memcpy(&mx, &scene[6], 4);
  ctx->bvh_eps = 1e-5f * mx;
  if (!(ctx->bvh_eps > 0.0f)) ctx->bvh_eps = 1e-30f;
  int32_t rc = sort_morton(ctx, n, keys, keys_tmp, ctx->bvh_order, order_tmp);
  if (rc != MNB_OK) return rc;
  const RayBvh t = ray_bvh(ctx, keys);
  MNB_LAUNCH(k_bvh_leaves, (n + 255) / 256, 256, 0, ctx->stream, (const float*)ctx->d_pos, (const uint32_t*)ctx->d_faces, t);
  if (n > 1) {
    MNB_LAUNCH(k_bvh_tree, (n - 1 + 255) / 256, 256, 0, ctx->stream, t);
    MNB_LAUNCH(k_bvh_refit, (n + 255) / 256, 256, 0, ctx->stream, t);
  }
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(ctx->stream));
  CK(ctx->d_ray_overflow.reserve(1));
  ctx->bvh_valid = true;
  return MNB_OK;
}

static int32_t ensure_raycaster(mnb_ctx* ctx) {
  if (ctx->bvh_valid) return MNB_OK;
  if (!ctx->V || !ctx->F) { ctx->err = "ray casting needs a mesh with faces"; return MNB_E_STATE; }
  const int32_t rc = build_raycaster(ctx);
  if (rc != MNB_OK) free_raycaster(ctx);       // no partial tree for the next call to allocate over
  return rc;
}

static int32_t check_ray_overflow(mnb_ctx* ctx) {
  unsigned int ov = 0;
  CK(cudaMemcpyAsync(&ov, ctx->d_ray_overflow, sizeof(ov), cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  if (ov) { ctx->err = "ray traversal stack exhausted (degenerate face distribution)"; return MNB_E_STATE; }
  return MNB_OK;
}

// staging of host-pointer inputs / outputs of the ray calls (floats)
static int32_t ensure_ray_io(mnb_ctx* ctx, size_t n_in, size_t n_out) {
  CK(ctx->d_ray_in.reserve(n_in)); CK(ctx->d_ray_out.reserve(n_out));
  return MNB_OK;
}

static int32_t impl_cast_rays(mnb_ctx* ctx, uint32_t n, const float* origins, const float* dirs, uint32_t dir_stride,
                              uint8_t* out_hit, float* out_dist, uint32_t* out_face, float* out_point) {
  if (!ctx || !ctx->V || (n && (!origins || !dirs)) || (dir_stride != 0 && dir_stride != 3)) return MNB_E_ARG;
  CK(cudaSetDevice(ctx->device));
  int32_t rc = ensure_raycaster(ctx);
  if (rc != MNB_OK) return rc;
  ctx->stats = mnb_stats{};
  if (!n) return MNB_OK;
  CallerArrays io(ctx);
  const size_t nd = dir_stride ? 3 * (size_t)n : 3;
  // staging layout (floats): in = origins[3n] dirs[nd]; out = dist[n] face[n] point[3n] hit[n bytes]
  if ((rc = ensure_ray_io(ctx, io.device() ? 0 : 3 * (size_t)n + nd, io.device() ? 0 : 6 * (size_t)n)) != MNB_OK) return rc;
  float* const st_in = ctx->d_ray_in; float* const st_out = ctx->d_ray_out;
  const float* const d_o = io.in(origins, st_in, 3 * (size_t)n);
  const float* const d_d = io.in(dirs, st_in + 3 * (size_t)n, nd);
  float* const d_dist = io.out(out_dist, st_out, n);
  uint32_t* const d_face = io.out(out_face, (uint32_t*)(st_out + n), n);
  float* const d_point = io.out(out_point, st_out + 2 * (size_t)n, 3 * (size_t)n);
  uint8_t* const d_hit = io.out(out_hit, (uint8_t*)(st_out + 5 * (size_t)n), n);
  CK(io.status());
  CK(cudaMemsetAsync(ctx->d_ray_overflow, 0, sizeof(unsigned int), ctx->stream));
  CK(cudaEventRecord(ctx->ev0, ctx->stream));
  MNB_LAUNCH(k_cast_rays, (n + 127) / 128, 128, 0, ctx->stream, ray_bvh(ctx), (const float*)ctx->d_pos, (const uint32_t*)ctx->d_faces, n,
             d_o, d_d, dir_stride, d_hit, d_dist, d_face, d_point, ctx->d_ray_overflow);
  CK(cudaGetLastError());
  CK(cudaEventRecord(ctx->ev1, ctx->stream));
  CK(io.copy_back());
  if ((rc = check_ray_overflow(ctx)) != MNB_OK) return rc;
  simple_stats(ctx, 1, n);
  return MNB_OK;
}

static int32_t impl_obstacle_reset(mnb_ctx* ctx) {
  if (!ctx || !ctx->V) return MNB_E_ARG;
  CK(cudaSetDevice(ctx->device));
  if (ctx->d_obst_mask) CK(cudaMemsetAsync(ctx->d_obst_mask, 0, (size_t)ctx->V, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return MNB_OK;
}

static int32_t impl_obstacle_update(mnb_ctx* ctx, uint32_t n_points, const float* points, const mnb_obstacle_params* P,
                                    uint32_t* out_lethals, uint32_t* n_lethals, uint32_t* out_changed, uint32_t* n_changed,
                                    float* out_costs) {
  if (!ctx || !ctx->V || !P || (n_points && !points) || !n_lethals || !n_changed) return MNB_E_ARG;
  CK(cudaSetDevice(ctx->device));
  int32_t rc = ensure_raycaster(ctx);
  if (rc != MNB_OK) return rc;
  const size_t V = ctx->V;
  CallerArrays io(ctx);
  const uint32_t n_tiles = (uint32_t)((V + US_TILE - 1) / US_TILE);
  if (!ctx->d_obst_mask) {
    CK(ctx->d_obst_now.reserve(V)); CK(ctx->d_obst_mask.reserve(V)); CK(ctx->d_obst_member.reserve(V));
    CK(ctx->d_obst_member_chg.reserve(V)); CK(ctx->d_obst_list.reserve(2 * V));
    CK(cudaMemsetAsync(ctx->d_obst_mask, 0, V, ctx->stream));
  }
  CK(ctx->d_changed.reserve(V)); CK(ctx->d_tile_count.reserve(n_tiles)); CK(ctx->d_total.reserve(1));
  if ((rc = ensure_ray_io(ctx, io.device() ? 0 : 3 * (size_t)n_points, (!io.device() && out_costs) ? V : 0)) != MNB_OK) return rc;
  const float* const d_pts = n_points ? io.in(points, ctx->d_ray_in.p, 3 * (size_t)n_points) : points;
  // the lists are produced without the caller's arrays too (the two halves of d_obst_list); their lengths are read back
  unsigned int totals[2] = {0, 0};
  uint32_t* const d_le = io.needed(out_lethals, ctx->d_obst_list.p, 1, &totals[0]);
  uint32_t* const d_ch = io.needed(out_changed, ctx->d_obst_list + V, 1, &totals[1]);
  float* const d_costs = io.out(out_costs, ctx->d_ray_out.p, V);
  CK(io.status());
  ObstacleArgs a{};
  for (int k = 0; k < 12; ++k) a.tf[k] = P->tf[k];
  for (int k = 0; k < 3; ++k) a.axis[k] = P->down_axis[k];
  a.max_obstacle_dist = P->max_obstacle_dist; a.robot_height = P->robot_height;
  CK(cudaMemsetAsync(ctx->d_obst_now, 0, V, ctx->stream));
  CK(cudaMemsetAsync(ctx->d_ray_overflow, 0, sizeof(unsigned int), ctx->stream));
  CK(cudaEventRecord(ctx->ev0, ctx->stream));
  if (n_points)
    MNB_LAUNCH(k_obstacle_rays, (n_points + 127) / 128, 128, 0, ctx->stream, ray_bvh(ctx), (const float*)ctx->d_pos, (const uint32_t*)ctx->d_faces,
               n_points, d_pts, a, ctx->d_obst_now, ctx->d_ray_overflow);
  MNB_LAUNCH(k_obstacle_diff, (unsigned)((V + 255) / 256), 256, 0, ctx->stream, ctx->V, (const uint8_t*)ctx->d_obst_now, ctx->d_obst_mask,
             ctx->d_obst_member, ctx->d_obst_member_chg, d_costs);
  for (int pass = 0; pass < 2; ++pass) {                   // ascending lists (std::set order): the new lethal set, the changed set
    const float* member = pass == 0 ? ctx->d_obst_member : ctx->d_obst_member_chg;
    MNB_LAUNCH(k_update_set_count, n_tiles, 256, 0, ctx->stream, member, (const float*)nullptr, ctx->V, ctx->d_tile_count);
    MNB_LAUNCH(k_update_set_scan, 1, 1024, 0, ctx->stream, ctx->d_tile_count, n_tiles, ctx->d_total);
    MNB_LAUNCH(k_update_set_write, n_tiles, 256, 0, ctx->stream, member, (const float*)nullptr, ctx->V, (const unsigned int*)ctx->d_tile_count,
               pass == 0 ? d_le : d_ch);
    CK(cudaMemcpyAsync(&totals[pass], ctx->d_total, sizeof(unsigned int), cudaMemcpyDeviceToHost, ctx->stream));
  }
  CK(cudaGetLastError());
  CK(cudaEventRecord(ctx->ev1, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  *n_lethals = totals[0]; *n_changed = totals[1];
  CK(io.copy_back());
  if ((rc = check_ray_overflow(ctx)) != MNB_OK) return rc;
  simple_stats(ctx, (n_points ? 1 : 0) + 7, n_points);
  return MNB_OK;
}

static int32_t impl_normal_clearance(mnb_ctx* ctx, const float* vertex_normals, float* out_clearance) {
  if (!ctx || !ctx->V || !out_clearance) return MNB_E_ARG;
  CK(cudaSetDevice(ctx->device));
  int32_t rc = ensure_raycaster(ctx);
  if (rc != MNB_OK) return rc;
  const size_t V = ctx->V;
  CallerArrays io(ctx);
  if ((rc = ensure_ray_io(ctx, (!io.device() && vertex_normals) ? 3 * V : 0, io.device() ? 0 : V)) != MNB_OK) return rc;
  const float* const d_vn = vertex_normals ? io.in(vertex_normals, ctx->d_ray_in.p, 3 * V) : ctx->d_vertex_normals.p;
  float* const d_out = io.out(out_clearance, ctx->d_ray_out.p, V);
  CK(io.status());
  CK(cudaMemsetAsync(ctx->d_ray_overflow, 0, sizeof(unsigned int), ctx->stream));
  CK(cudaEventRecord(ctx->ev0, ctx->stream));
  MNB_LAUNCH(k_normal_clearance, (unsigned)((V + 127) / 128), 128, 0, ctx->stream, ray_bvh(ctx), (const float*)ctx->d_pos, (const uint32_t*)ctx->d_faces,
             ctx->V, d_vn, d_out, ctx->d_ray_overflow);
  CK(cudaGetLastError());
  CK(cudaEventRecord(ctx->ev1, ctx->stream));
  CK(io.copy_back());
  if ((rc = check_ray_overflow(ctx)) != MNB_OK) return rc;
  simple_stats(ctx, 1, ctx->V);
  return MNB_OK;
}

extern "C" {
int32_t mnb_cast_rays(mnb_ctx* ctx, uint32_t n, const float* origins, const float* dirs, uint32_t dir_stride, uint8_t* out_hit,
                      float* out_dist, uint32_t* out_face, float* out_point) {
  return guarded(ctx, [&]() { return impl_cast_rays(ctx, n, origins, dirs, dir_stride, out_hit, out_dist, out_face, out_point); });
}
int32_t mnb_obstacle_update(mnb_ctx* ctx, uint32_t n_points, const float* points, const mnb_obstacle_params* params,
                            uint32_t* out_lethals, uint32_t* n_lethals, uint32_t* out_changed, uint32_t* n_changed, float* out_costs) {
  return guarded(ctx, [&]() { return impl_obstacle_update(ctx, n_points, points, params, out_lethals, n_lethals, out_changed, n_changed, out_costs); });
}
int32_t mnb_obstacle_reset(mnb_ctx* ctx) { return guarded(ctx, [&]() { return impl_obstacle_reset(ctx); }); }
int32_t mnb_normal_clearance(mnb_ctx* ctx, const float* vertex_normals, float* out_clearance) {
  return guarded(ctx, [&]() { return impl_normal_clearance(ctx, vertex_normals, out_clearance); });
}
}  // extern "C"
