/*
 * meshnav_b200.h -- C ABI of libmeshnav_b200.so
 *
 * H100-native (sm_90a CUDA) replacement for the wavefront hot path of
 * naturerobots/mesh_navigation.  Plain pointers and sizes only; no C++ / torch
 * types cross this boundary.  Every entry point names the reference interface
 * it stands in for (paths relative to the reference repo).
 *
 * Conventions
 *   - all calls return MNB_OK (0) or a negative MNB_E_* code, except the
 *     planner calls which return the MBF GetPath::Result code the reference's
 *     makePlan would return (dijkstra_mesh_planner.h:72-85): 0 SUCCESS,
 *     51 CANCELED, 52 INVALID_START, 53 INVALID_GOAL, 54 NO_PATH_FOUND,
 *     or a negative MNB_E_* code on CUDA / argument errors.
 *   - array arguments are HOST pointers by default.  After
 *     mnb_set_pointer_mode(ctx, MNB_PTR_DEVICE) array arguments of the
 *     per-call functions (costs, weights, outputs) are DEVICE pointers on the
 *     context's device and no host<->device copy happens inside the call.
 *   - the library never frees or keeps caller memory; outputs are written into
 *     caller-provided buffers of the stated length.
 *   - an mnb_ctx is single-caller (one stream); mnb_cancel() is the only entry
 *     point that may be called concurrently from another thread
 *     (reference: CVPMeshPlanner::cancel, cvp_mesh_planner.cpp:142-146).
 *   - there is NO CPU fallback: every compute entry point fails with
 *     MNB_E_CUDA if no sm_90 device is usable.
 */
#ifndef MESHNAV_B200_H
#define MESHNAV_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MNB_OK 0
#define MNB_E_ARG (-1)
#define MNB_E_CUDA (-2)
#define MNB_E_STATE (-3)
#define MNB_E_NCCL (-4)
#define MNB_E_NOMEM (-5)

/* MBF outcome codes (mbf_msgs/action/GetPath; dijkstra_mesh_planner.h:72-85) */
#define MNB_SUCCESS 0
#define MNB_CANCELED 51
#define MNB_INVALID_START 52
#define MNB_INVALID_GOAL 53
#define MNB_NO_PATH_FOUND 54

#define MNB_PTR_HOST 0
#define MNB_PTR_DEVICE 1

typedef struct mnb_ctx mnb_ctx;

/* ---- lifetime ----------------------------------------------------------- */
int32_t mnb_create(int32_t device, mnb_ctx** out_ctx);
void mnb_destroy(mnb_ctx* ctx);
const char* mnb_last_error(mnb_ctx* ctx);
int32_t mnb_set_pointer_mode(mnb_ctx* ctx, int32_t mode);
/* cudaStream_t (as void*) the context launches on; lets a caller time with CUDA events. */
void* mnb_stream(mnb_ctx* ctx);

/* ---- map upload: replaces the lvr2 half-edge mesh the plugins read ------
 * mesh_map::MeshMap::mesh() / edgeDistances() (mesh_map.h:97-452, mesh_map.cpp:404-425).
 * pos[3V] float xyz, faces[3F] vertex ids in the mesh's cyclic (CCW) order.
 * edges[2E] may be NULL: the library then numbers edges by ascending (lo,hi)
 * vertex pair; pass the caller's own edge order (e.g. lvr2 EdgeHandle order)
 * so that edge_weights / edge_distances arrays use the caller's indices.
 * Always HOST pointers (one-time setup). */
int32_t mnb_set_mesh(mnb_ctx* ctx, uint32_t V, uint32_t F, const float* pos, const uint32_t* faces,
                     const uint32_t* edges, uint32_t E);
uint32_t mnb_num_vertices(mnb_ctx* ctx);
uint32_t mnb_num_faces(mnb_ctx* ctx);
uint32_t mnb_num_edges(mnb_ctx* ctx);
int32_t mnb_get_edges(mnb_ctx* ctx, uint32_t* out_edges /* 2E, host */);
/* lvr2::calcVertexDistances as used for MeshMap::edge_distances (mesh_map.cpp:414) */
int32_t mnb_get_edge_distances(mnb_ctx* ctx, float* out_edge_distances /* E */);

/* ---- MeshMap::computeEdgeWeights (mesh_map.cpp:517-561) -----------------
 * edge_weights[e] = +inf if an endpoint cost is inf, else
 * dist[e] + edge_cost_factor * (dist[e] * (c1 + c2) / 2).  Writes out_edge_weights (E) if
 * non-NULL and installs vertex_costs + the weights as the planners' inputs. */
int32_t mnb_compute_edge_weights(mnb_ctx* ctx, const float* vertex_costs /* V */, double edge_cost_factor,
                                 float* out_edge_weights /* E or NULL */);

/* ---- per-plan inputs the planners read from the map ---------------------
 * MeshMap::vertexCosts() / edgeWeights() / invalid
 * (cvp_mesh_planner.cpp:245,663-664; dijkstra_mesh_planner.cpp:214,227-229).
 * invalid may be NULL (no invalid vertices). */
int32_t mnb_set_costs(mnb_ctx* ctx, const float* vertex_costs /* V */, const float* edge_weights /* E */,
                      const uint8_t* invalid /* V or NULL */);

/* ---- DijkstraMeshPlanner::dijkstra (dijkstra_mesh_planner.cpp:217-398) ---
 * seed_vertex  = the reference's start_vertex (nearest vertex to the navigation goal, :235)
 * robot_vertex = the reference's goal_vertex (nearest vertex to the robot, :236) or -1 for a
 *                full field.  out_dist[V] (+inf = unreached), out_pred[V] (self = none). */
int32_t mnb_dijkstra(mnb_ctx* ctx, uint32_t seed_vertex, int64_t robot_vertex, double cost_limit,
                     double goal_dist_offset, float* out_dist, uint32_t* out_pred);

/* Batched full-field Dijkstra: n independent DijkstraMeshPlanner::dijkstra waves (dijkstra_mesh_planner.cpp:217-398,
 * robot vertex -1) on the installed map, hundreds of them in flight at once.  Row k of out_dist / out_pred ([n][V]
 * row-major) is the field seeded at seed_vertices[k], bit-identical to mnb_dijkstra(ctx, seed_vertices[k], -1,
 * cost_limit, ...): +inf / self where unreached.  Either output may be NULL, not both; duplicate seeds are allowed.
 * A predecessor row is the whole shortest-path tree towards its seed: walking pred from any vertex gives its path.
 * seed_vertices is always a host pointer; the outputs follow mnb_set_pointer_mode.  MNB_INVALID_START if a seed is
 * >= V (checked before anything is written).  The number of concurrent waves is capped by the free device memory
 * (16 bytes per vertex and wave), so a large map runs with fewer of them.  The waves use a workspace of their own: the
 * results of the last mnb_cvp (mnb_cvp_backtrack, mnb_vector_map with pred = NULL) and of the last inflation
 * (mnb_inflation_vector_map) remain available after this call. */
int32_t mnb_dijkstra_batch(mnb_ctx* ctx, uint32_t n, const uint32_t* seed_vertices /* n, host */, double cost_limit,
                           float* out_dist /* [n][V] or NULL */, uint32_t* out_pred /* [n][V] or NULL */);

/* ---- CVPMeshPlanner::waveFrontPropagation (cvp_mesh_planner.cpp:651-886) -
 * seed_face / seed_pos = the reference's start_face / start (navigation goal, :673,:719-728)
 * robot_face           = the reference's goal_face (:674) or -1 for a full field.
 * Outputs (any may be NULL): potential_ , predecessors_, direction_, cutting_faces_ (-1 = none). */
int32_t mnb_cvp(mnb_ctx* ctx, uint32_t seed_face, const float seed_pos[3], int64_t robot_face,
                double cost_limit, double goal_dist_offset, float* out_dist, uint32_t* out_pred,
                float* out_direction, int32_t* out_cutting_face);

/* CVP replanning after cost updates: the outputs and the return code are bit-identical to mnb_cvp with the same
 * arguments on the currently installed costs.  changed (n_changed entries, always a host pointer, any order, duplicates
 * and unchanged vertices allowed) is the union of the changed sets of the mnb_update_vertex_costs calls since the last
 * successful mnb_cvp_replan on this context; the caller keeps it, as for mnb_dijkstra_batch_repair.
 * The context keeps the wave of the last successful replan in a workspace of its own (about 44 bytes per vertex plus the
 * level pool, allocated by the first call).  When seed_face, the bits of seed_pos and of cost_limit are those of that
 * wave and the costs changed since only through mnb_update_vertex_costs, the wave resumes from the earliest pop time the
 * change can reach -- the earliest pop among the changed vertices and their face neighbours, the moment the old goal
 * cutoff armed, or the moment the new robot face's vertices had all popped -- and re-runs only what comes after it;
 * robot_face and goal_dist_offset may differ.  Otherwise (also after mnb_set_costs / mnb_compute_edge_weights / a cancelled
 * call, when that moment is not after every seed's pop, or when the level pool lacks room) it runs one whole wave.
 * mnb_get_stats counts the resumed part only (rounds, recomputes, settled).  mnb_cvp, the batch calls, the matrices,
 * the field repair and the inflation calls may run between two replans without disturbing the resident wave.  On success
 * the result is the last plan for mnb_cvp_backtrack and mnb_vector_map (pred = NULL), as after mnb_cvp.  Nothing is
 * written on MNB_E_ARG (a changed id >= V, a NULL array that is needed), MNB_E_STATE (no costs), MNB_INVALID_START /
 * MNB_INVALID_GOAL (as mnb_cvp).  mnb_cancel: MNB_CANCELED, and the next call runs a whole wave.  The outputs follow
 * mnb_set_pointer_mode and may be NULL. */
int32_t mnb_cvp_replan(mnb_ctx* ctx, uint32_t seed_face, const float seed_pos[3], int64_t robot_face,
                       double cost_limit, double goal_dist_offset, uint32_t n_changed, const uint32_t* changed /* host */,
                       float* out_dist, uint32_t* out_pred, float* out_direction, int32_t* out_cutting_face);

/* Batched full-field CVP potentials: n independent goals on the installed map, one wavefront
 * per thread-block cluster, all SMs busy.  out_dist is [n][V] row-major.  Same call as mnb_cvp_batch_fields with
 * out_dist alone: the number of concurrent waves is capped by the free device memory as well. */
int32_t mnb_cvp_batch(mnb_ctx* ctx, uint32_t n, const uint32_t* seed_faces /* n, host */,
                      const float* seed_pos /* 3n, host */, double cost_limit, float* out_dist);

/* Batched full-field CVP vector fields: n independent goals, like mnb_cvp_batch, with the inputs of the vector field as
 * well.  Row k of each output ([n][V] row-major) is bit-identical to the same output of mnb_cvp(ctx, seed_faces[k],
 * &seed_pos[3k], -1, cost_limit, ...): potential (+inf = unreached), predecessor (self = none), direction (0 = none)
 * and cutting face (-1 = none; a seed vertex has itself, 0 and the seed face).  Any output may be NULL, not all of them;
 * duplicate goals are allowed.  Rows k of pred / direction / cutting face feed mnb_vector_map(ctx, pred_k, dir_k,
 * cut_k, out), which is CVPMeshPlanner::computeVectorMap (cvp_mesh_planner.cpp:204-239): one vector field per goal,
 * e.g. one per robot of a fleet.  seed_faces / seed_pos are always host pointers; the outputs follow
 * mnb_set_pointer_mode.  MNB_INVALID_START if a seed face is >= F (checked before anything is written); MNB_CANCELED
 * after mnb_cancel (the rows are then incomplete).  With out_dist alone the call is mnb_cvp_batch; with any
 * other output each wave derives its rows before it takes the next goal.  The number of concurrent waves is capped by the free
 * device memory (~64 bytes per vertex and wave) as well as by the CTA slots, so a large map runs with fewer of them;
 * MNB_E_NOMEM if not even one fits.  The waves share the wavefront workspace with mnb_cvp and the inflation wave: the
 * last inflation's labels are dropped (as after mnb_cvp_batch), while the outputs of the last mnb_cvp
 * (mnb_cvp_backtrack, mnb_vector_map with pred = NULL) remain available. */
int32_t mnb_cvp_batch_fields(mnb_ctx* ctx, uint32_t n, const uint32_t* seed_faces /* n, host */,
                             const float* seed_pos /* 3n, host */, double cost_limit,
                             float* out_dist /* [n][V] or NULL */, uint32_t* out_pred /* [n][V] or NULL */,
                             float* out_direction /* [n][V] or NULL */, int32_t* out_cutting_face /* [n][V] or NULL */);

/* Batched CVP replanning after cost updates: the fleet's vector fields kept up to date without running every goal's wave
 * again.  The outputs and the return code are bit-identical to mnb_cvp_batch_fields(ctx, n, seed_faces, seed_pos,
 * cost_limit, ...) on the currently installed costs.  Any output may be NULL, not all of them.
 * changed (n_changed entries, always a host pointer, any order, duplicates and unchanged vertices allowed) is the union
 * of the changed sets of the mnb_update_vertex_costs calls since the last successful mnb_cvp_batch_replan on this
 * context; the caller keeps it, as for mnb_cvp_replan.
 * The context keeps a store of resident waves keyed by goal (seed face and the bits of the seed position).  A goal of
 * this call resumes from its own T0 -- the earliest old pop time among the changed vertices and their face neighbours --
 * when its wave is resident, the bits of cost_limit and the costs are those of the store (only mnb_update_vertex_costs
 * since), its level pool is at most half full and every seed vertex pops before T0.  Any other goal runs a whole wave,
 * which becomes resident if a slot is free.  Goals may be added, dropped or reordered between calls (matching is by
 * key); resident goals absent from a call are released; duplicate goals share one wave and their rows are copies.
 * A resident goal costs about 44 bytes per vertex (label, side arrays, level pool, pred / direction / cutting-face rows);
 * the number of slots is capped by the device memory left after the workspace of the concurrent waves, and goals past
 * the cap run whole waves on every call, still exact.  A resumed wave that overflows its level pool runs again as a
 * whole wave.  mnb_get_stats sums rounds, recomputes and settled over the waves (a resumed goal counts its re-run tail).
 * Nothing is written on MNB_E_ARG (n == 0, a NULL array that is needed, a changed id >= V), MNB_E_STATE (no costs),
 * MNB_INVALID_START (a seed face >= F), MNB_E_NOMEM (not even one concurrent wave fits).  mnb_cancel: MNB_CANCELED,
 * the rows are incomplete, the store is dropped and the next call runs whole waves.  mnb_set_mesh frees the store;
 * mnb_set_costs and mnb_compute_edge_weights make it stale.  No other call disturbs it, and it disturbs neither
 * mnb_cvp_replan's resident wave nor the last mnb_cvp result (mnb_cvp_backtrack, mnb_vector_map); it shares the
 * wavefront workspace as mnb_cvp_batch_fields does, so the last inflation's labels are dropped.  The outputs follow
 * mnb_set_pointer_mode. */
int32_t mnb_cvp_batch_replan(mnb_ctx* ctx, uint32_t n, const uint32_t* seed_faces /* n, host */,
                             const float* seed_pos /* 3n, host */, double cost_limit,
                             uint32_t n_changed, const uint32_t* changed /* host */,
                             float* out_dist /* [n][V] or NULL */, uint32_t* out_pred /* [n][V] or NULL */,
                             float* out_direction /* [n][V] or NULL */, int32_t* out_cutting_face /* [n][V] or NULL */);
/* Frees the resident store of mnb_cvp_batch_replan (it can reach tens of GB); the next call runs whole waves. */
int32_t mnb_cvp_batch_replan_release(mnb_ctx* ctx);

/* Cost matrices: the cost from each of n seeds to each of m target vertices, e.g. from every candidate goal to every
 * robot of a fleet, without the [n][V] rows.  out[k][j] ([n][m] row-major) is bit-identical to
 * dist[k][target_vertices[j]] of mnb_dijkstra_batch (mnb_dijkstra_matrix) or of mnb_cvp_batch (mnb_cvp_matrix) with
 * the same seeds and cost_limit: +inf where the target is unreached.  A wave stops as soon as every target has
 * settled -- its label is then final -- so targets near their seeds cost a fraction of the full field; mnb_get_stats
 * reports the settled vertices and rounds summed over the waves.  Duplicate seeds and duplicate targets are allowed.
 * The seed and target arrays are always host pointers; out follows mnb_set_pointer_mode.  Errors, with nothing
 * written: MNB_E_ARG for n == 0, m == 0 or a NULL array; MNB_E_STATE without costs; MNB_INVALID_START for a seed
 * >= V (Dijkstra) or a seed face >= F (CVP); MNB_INVALID_GOAL for a target >= V.  MNB_CANCELED after mnb_cancel: no
 * new goal is taken once the flag is set (the matrix is then incomplete).  No [n][V] rows are allocated in either
 * pointer mode; the number of concurrent waves is capped as for the batch calls, by the workspace alone.
 * mnb_dijkstra_matrix runs in mnb_dijkstra_batch's workspace: the results of the last mnb_cvp and of the last
 * inflation stay available.  mnb_cvp_matrix shares the wavefront workspace like mnb_cvp_batch: the last inflation's
 * labels are dropped, the outputs of the last mnb_cvp remain available. */
int32_t mnb_dijkstra_matrix(mnb_ctx* ctx, uint32_t n, const uint32_t* seed_vertices /* n, host */,
                            uint32_t m, const uint32_t* target_vertices /* m, host */, double cost_limit,
                            float* out /* [n][m] */);
int32_t mnb_cvp_matrix(mnb_ctx* ctx, uint32_t n, const uint32_t* seed_faces /* n, host */, const float* seed_pos /* 3n, host */,
                       uint32_t m, const uint32_t* target_vertices /* m, host */, double cost_limit,
                       float* out /* [n][m] */);

/* Dijkstra field repair: brings resident distance and predecessor rows up to date after cost updates by re-running only
 * the region the change can reach.  On entry row k of io_dist / io_pred ([n][V] row-major) is the field of
 * mnb_dijkstra_batch(seed_vertices[k], cost_limit) -- or, the same thing, of a full-field mnb_dijkstra (robot vertex
 * -1) -- computed on the costs installed before one or more mnb_update_vertex_costs calls, and changed[n_changed] holds
 * the union of those calls' changed sets (any order, duplicates and vertices whose cost did not change allowed).  On
 * return row k is bit-identical to mnb_dijkstra_batch on the current costs, predecessors included.
 * The caller is responsible for the changed set: a vertex left out of it leaves its region stale.  mnb_set_costs or
 * mnb_compute_edge_weights between the rows and the repair invalidate the rows unless every vertex is passed as changed.
 * Work: the vertices whose predecessor chain runs through a changed vertex are reset and re-reached, the rest keep their
 * labels unless the change lowers them.  mnb_get_stats reports rounds, recomputes and settled vertices summed over the
 * waves, as for mnb_dijkstra_batch.  seed_vertices and changed are host pointers; the rows follow mnb_set_pointer_mode:
 * device rows are repaired in place, host rows are uploaded and downloaded.  n_changed == 0 returns MNB_SUCCESS and
 * leaves the rows untouched.  Errors, with nothing written: MNB_E_ARG for n == 0, a NULL array or a changed vertex >= V;
 * MNB_E_STATE without costs; MNB_INVALID_START for a seed >= V.  MNB_CANCELED after mnb_cancel: the rows are then not
 * valid, and the caller recomputes them (mnb_dijkstra_batch).  Runs in mnb_dijkstra_batch's workspace, under the same
 * memory cap: the results of the last mnb_cvp and of the last inflation stay available. */
int32_t mnb_dijkstra_batch_repair(mnb_ctx* ctx, uint32_t n, const uint32_t* seed_vertices /* n, host */, double cost_limit,
                                  uint32_t n_changed, const uint32_t* changed /* n_changed, host */,
                                  float* io_dist /* [n][V] */, uint32_t* io_pred /* [n][V] */);

/* ---- InflationLayer::waveCostInflation (inflation_layer.cpp:341-491) -----
 * lethals[n] (any order, duplicates allowed).  Uses edge_distances (:383), not edge_weights.
 * out_dist[V]: distances_ (+inf = not in the sparse map); out_cost[V]: riskiness_ =
 * fading(dist) (NaN = not in the sparse map).  Either may be NULL. */
typedef struct mnb_inflation_params {
  double inscribed_radius;    /* 0.25  (inflation_layer.h:240-248) */
  double inflation_radius;    /* 0.4  */
  double lethal_value;        /* 1.0  */
  double inscribed_value;     /* 0.99 */
  double cost_scaling_factor; /* 1.0  */
} mnb_inflation_params;
int32_t mnb_inflate(mnb_ctx* ctx, const uint32_t* lethals, uint32_t n, const uint8_t* invalid /* V or NULL */,
                    const mnb_inflation_params* params, float* out_dist, float* out_cost);

/* ---- geometric cost layers + MaxCombinationLayer (mesh_layers/src/<name>_layer.cpp) -------------------
 * HeightDiffLayer::computeLayer (height_diff_layer.cpp:103-110), RoughnessLayer (roughness_layer.cpp:91-147),
 * SteepnessLayer (steepness_layer.cpp:100-170), RidgeLayer (ridge_layer.cpp:101-187), ClearanceLayer cost
 * mapping (clearance_layer.cpp:67-99, on a caller-provided clearance array; NULL = +inf, no ray hits),
 * BorderLayer (border_layer.cpp:104-110), computeLethals (cost > threshold) and
 * MaxCombinationLayer::computeLayer (combination_layer.cpp:44-85), fused into ONE per-vertex kernel.
 * out_costs: 6*V floats, layer-major in the order height_diff, roughness, steepness, ridge, clearance,
 * border; out_combined: V; out_lethal_mask: V bytes, bit i = lethal in layer i.  Any output may be NULL;
 * the results also stay resident on the device for chaining. */
typedef struct mnb_layer_params {
  double height_diff_threshold, height_diff_radius;           /* 0.185, 0.3 */
  double roughness_threshold, roughness_radius;               /* 0.3, 0.3 */
  double steepness_threshold;                                 /* 0.3 */
  double ridge_threshold, ridge_radius;                       /* 0.3, 0.3 */
  double clearance_robot_height, clearance_height_inflation;  /* 0.5, 0.3 */
  double border_threshold, border_cost;                       /* 0.5, 1.0 */
} mnb_layer_params;
int32_t mnb_compute_layers(mnb_ctx* ctx, const mnb_layer_params* params, const float* clearance /* V or NULL */,
                           float* out_costs, float* out_combined, uint8_t* out_lethal_mask);
/* lvr2::calcVertexNormals equivalent (mesh_map.cpp:374): normalised sum of incident face normals */
int32_t mnb_get_vertex_normals(mnb_ctx* ctx, float* out_normals /* 3V */);

/* ---- localisation -----------------------------------------------------------------------------------
 * MeshMap::getNearestVertexHandle (mesh_map.cpp:1161-1174) and MeshMap::searchContainingFace / getContainingFace
 * (mesh_map.cpp:1110-1159) for n query points at once: out_vertex[q] = nearest vertex (exhaustive, ties to the lowest
 * id), out_face[q] = the incident face of that vertex containing the projected point (-1: none), out_bary its
 * barycentric coordinates.  Any of the outputs may be NULL. */
int32_t mnb_locate(mnb_ctx* ctx, uint32_t n, const float* points /* 3n */, uint32_t* out_vertex /* n */,
                   int32_t* out_face /* n */, float* out_bary /* 3n */);

/* ---- vector-field epilogues -----------------------------------------------------------------------
 * DijkstraMeshPlanner::computeVectorMap (dijkstra_mesh_planner.cpp:189-209): direction == NULL, cutting_face == NULL:
 *   out[v] = normalize(p[pred[v]] - p[v]).
 * CVPMeshPlanner::computeVectorMap (cvp_mesh_planner.cpp:204-239): the vector is additionally rotated about the vertex
 *   normal by direction[v]; vertices without a cutting face are skipped.
 * out_vec: 3V floats, NaN = "no entry in the sparse vector map" (pred[v] == v or no cutting face).
 * pred == NULL: the field of the LAST successful mnb_cvp on this context, from its device-resident result (nothing is uploaded). */
int32_t mnb_vector_map(mnb_ctx* ctx, const uint32_t* pred /* V or NULL */, const float* direction /* V or NULL */,
                       const int32_t* cutting_face /* V or NULL */, float* out_vec /* 3V */);

/* ---- vector-field back-tracking -------------------------------------------------------------------
 * The tail of CVPMeshPlanner::waveFrontPropagation (cvp_mesh_planner.cpp:920-951): follows the vector field of the
 * LAST successful mnb_cvp on this context (kept on the device) from the robot position down to the wave's seed with
 * MeshMap::meshAhead (mesh_map.cpp:1070-1108) in steps of step_width.  Points are returned in walk order
 * (robot first, seed last = the order of the final plan after cvp:100 path.reverse()).  In device-pointer mode
 * the result arrays of that mnb_cvp must still be alive.  Layer vector fields (AbstractLayer::vectorAt) are zero.
 * Returns MNB_SUCCESS / MNB_NO_PATH_FOUND / MNB_CANCELED; MNB_E_STATE if max_points is exhausted. */
int32_t mnb_cvp_backtrack(mnb_ctx* ctx, const float robot_pos[3], uint32_t robot_face, double step_width, uint32_t max_points,
                          float* path_pos /* 3*max_points */, uint32_t* path_face /* max_points or NULL */,
                          uint32_t* n_points);

/* ---- incremental updates: the sensor-rate callers of the hot path (SURVEY.md 3.4) ----------------------------------
 * NaN marks "no entry" in a sparse lvr2 cost map; `changed` plays the std::set<VertexHandle> of the reference
 * (any order, duplicates allowed).  All three work on the changed vertices only. */

/* MeshMap::layerChanged (mesh_map.cpp:455-492) + MeshMap::updateEdgeWeights (mesh_map.cpp:563-618):
 *   vertex_costs[v] = cost_map.get(v).value_or(default_value) for v in changed, then the weights of the edges incident
 *   to a changed vertex are recomputed with the formula of computeEdgeWeights -- and, exactly as in the reference
 *   (:568-572), NOT AT ALL when edge_cost_factor == 0.  The planners' derived tables are refreshed for those edges only
 *   (no V- or E-sized pass, no re-upload).  costs_indexed_by_vertex == 0: costs[i] is the new cost of changed[i];
 *   != 0: costs is the layer's V-sized map and default_value replaces NaN entries.  Needs mnb_set_costs /
 *   mnb_compute_edge_weights first. */
int32_t mnb_update_vertex_costs(mnb_ctx* ctx, uint32_t n_changed, const uint32_t* changed, const float* costs,
                                int32_t costs_indexed_by_vertex, float default_value, double edge_cost_factor);
/* the installed per-plan inputs (MeshMap::vertexCosts() / edgeWeights()); either may be NULL */
int32_t mnb_get_costs(mnb_ctx* ctx, float* out_vertex_costs /* V */, float* out_edge_weights /* E */);

/* MaxCombinationLayer::onInputChanged (combination_layer.cpp:87-147) for the changed vertices:
 *   io_costs[v] = max(0, max_i (layer_costs[i][v] or defaults[i]));  io_lethal[v] = OR_i layer_lethal[i][v].
 * layer_costs / layer_lethal are HOST arrays of n_layers (<= 8) pointers to V-sized maps (host or device per the
 * pointer mode); layer_lethal, any of its entries and io_lethal may be NULL; defaults is a host array. */
int32_t mnb_max_combination_update(mnb_ctx* ctx, uint32_t n_layers, const float* const* layer_costs, const float* defaults,
                                   const uint8_t* const* layer_lethal, uint32_t n_changed, const uint32_t* changed,
                                   float* io_costs /* V */, uint8_t* io_lethal /* V or NULL */);

/* AvgCombinationLayer::onInputChanged / computeLayer (combination_layer.cpp:185-302) for the changed vertices:
 *   io_costs[v] = sum_i weights[i] * (layer_costs[i][v] or defaults[i]), accumulated in layer order in float;
 *   io_lethal[v] = OR_i layer_lethal[i][v].  weights = AbstractLayer::combinationWeight() of the inputs (host array). */
int32_t mnb_avg_combination_update(mnb_ctx* ctx, uint32_t n_layers, const float* const* layer_costs, const float* defaults,
                                   const float* weights, const uint8_t* const* layer_lethal, uint32_t n_changed,
                                   const uint32_t* changed, float* io_costs /* V */, uint8_t* io_lethal /* V or NULL */);

/* InflationLayer::onInputChanged (inflation_layer.cpp:97-179): re-runs waveCostInflation from `lethals` (the reference
 * does a full re-inflation here too, :143-151) and reports the update set handed to notifyChange (:154-176): the
 * vertices that carry a riskiness value now or carried one after the previous mnb_inflate / mnb_inflation_update on this
 * context, ascending.  out_changed: room for V ids (may be NULL); *n_changed (host) receives the count. */
int32_t mnb_inflation_update(mnb_ctx* ctx, const uint32_t* lethals, uint32_t n, const uint8_t* invalid /* V or NULL */,
                             const mnb_inflation_params* params, float* out_dist, float* out_cost,
                             uint32_t* out_changed /* V */, uint32_t* n_changed);

/* The same result from the part of the map a change can reach.  Arguments and pointer modes are those of
 * mnb_inflation_update (lethals: the whole new lethal set; duplicates and ids >= V are ignored as there); out_dist and
 * out_cost are bit-identical to what it returns.  out_changed (room for V ids, may be NULL) lists, ascending, exactly the
 * vertices whose riskiness entry changed against the previous inflation result on this context -- presence or value
 * bits, NaN = no entry, NaN equal to NaN -- which is the set to hand to mnb_max_combination_update /
 * mnb_update_vertex_costs; *n_changed (host) receives the count.
 * The previous result may come from mnb_inflate, mnb_inflation_update or an earlier repair, with planner calls in
 * between.  A cluster of that result (a connected component of its finite distances_, linked through shared faces) is
 * affected when it contains or shares a face with a vertex whose lethal or invalid flag changed; the wave re-runs from
 * the new lethals of the affected clusters and the new ones outside the old footprint, and again with more clusters while
 * its footprint touches an unaffected one; every other vertex keeps its bits (DESIGN §4).  Without a previous result, or
 * with params not bitwise equal to its params, one whole-map wave runs, and so it does when more than half of the old
 * footprint lies in affected clusters (the call chooses; the changed set is the same tight set).  An unchanged lethal set
 * and mask run no wave and leave the wave's labels in the workspace as they were.
 * A repulsive field made valid by mnb_inflation_vector_map stays valid: it is recomputed on the region, and
 * mnb_inflation_vector_map returns it.  Otherwise mnb_inflation_vector_map needs whole-map labels: it works after a
 * whole-map wave (and after a call that ran no wave, if it worked before it) and returns MNB_E_STATE after a local one.  Stats: rounds, recomputes and settled summed over the passes; each pass launches three kernels. */
int32_t mnb_inflation_repair(mnb_ctx* ctx, const uint32_t* lethals, uint32_t n, const uint8_t* invalid /* V or NULL */,
                             const mnb_inflation_params* params, float* out_dist /* V or NULL */, float* out_cost /* V or NULL */,
                             uint32_t* out_changed /* V or NULL */, uint32_t* n_changed /* host */);

/* ---- ray casting against the map -------------------------------------------------------------------------------------
 * The shared raycaster of the map (MeshMap::raycaster(), mesh_map.h:318; lvr2::EmbreeRaycaster / BVHRaycaster built at
 * mesh_map.cpp:317-321) as a linear BVH over the faces on the device, built at the first ray call after mnb_set_mesh.
 * Results are those of a loop over all faces (the tree only prunes): two-sided Moeller-Trumbore in float, nearest hit,
 * ties to the smallest face id -- the arithmetic is spelled out in oracle/oracle.cpp ("Ray casting against the map").
 *
 * mnb_cast_rays = RaycasterBase::castRays as called at obstacle_layer.cpp:239.  dirs: one unit vector per ray
 * (dir_stride 3) or one for all rays (dir_stride 0, obstacle_layer.cpp:229).  Outputs (each may be NULL): hit flag,
 * distance (+inf: no hit), face id (0xffffffff: no hit), hit point (NaN: no hit). */
int32_t mnb_cast_rays(mnb_ctx* ctx, uint32_t n, const float* origins /* 3n */, const float* dirs, uint32_t dir_stride,
                      uint8_t* out_hit /* n */, float* out_dist /* n */, uint32_t* out_face /* n */, float* out_point /* 3n */);

/* ObstacleLayer::processPointCloud (obstacle_layer.cpp:215-296) without the ROS plumbing: points are the cloud in the
 * message frame; tf the row-major 3x4 [R|t] of the message frame -> map frame transform (:176-180); down_axis the
 * configured axis already rotated into the map frame (:183-205).  Points with |p| <= max_obstacle_dist are transformed
 * and cast along down_axis; a hit within robot_height makes the three vertices of the hit face lethal (:245-256).
 * out_lethals: the new lethal set, ascending (lethals_); out_changed: its symmetric difference with the set of the
 * previous call on this context (:268-273, what notifyChange receives); both need room for V ids and may be NULL; the
 * counts go to the host.  out_costs (V floats or NULL): +inf on lethal vertices, NaN = no entry (costs_, :250;
 * defaultValue() 0).  mnb_obstacle_reset empties the remembered lethal set. */
typedef struct mnb_obstacle_params {
  double max_obstacle_dist, robot_height;
  float tf[12];
  float down_axis[3];
} mnb_obstacle_params;
int32_t mnb_obstacle_update(mnb_ctx* ctx, uint32_t n_points, const float* points /* 3n */, const mnb_obstacle_params* params,
                            uint32_t* out_lethals /* V */, uint32_t* n_lethals, uint32_t* out_changed /* V */,
                            uint32_t* n_changed, float* out_costs /* V or NULL */);
int32_t mnb_obstacle_reset(mnb_ctx* ctx);

/* lvr2::calcNormalClearance (clearance_layer.cpp:161): the free space above every vertex = distance along its normal
 * to the first face not incident to it, +inf if there is none; the input of the clearance cost mapping of
 * mnb_compute_layers.  vertex_normals: 3V floats or NULL = the normals mnb_set_mesh computed. */
int32_t mnb_normal_clearance(mnb_ctx* ctx, const float* vertex_normals, float* out_clearance /* V */);

/* ---- InflationLayer repulsive vector field -------------------------------------------------------------------------
 * vector_map_ as InflationLayer::waveFrontUpdate accumulates it (inflation_layer.cpp:277-308) for the LAST mnb_inflate /
 * mnb_inflation_update on this context; zero = no entry.  Derived from that wave's final labels, which live in the
 * workspace the planners share: call it before the next planner call on the context (MNB_E_STATE otherwise).  The field
 * and distances_ stay resident on the device.  out_vectors (3V) may be NULL. */
int32_t mnb_inflation_vector_map(mnb_ctx* ctx, float* out_vectors);
/* InflationLayer::vectorAt(vertices, barycentric_coords) (inflation_layer.cpp:493-521) of the resident field for n samples:
 * faces_q[n] face ids, bary[3n] -> out[3n]. */
int32_t mnb_inflation_vector_at(mnb_ctx* ctx, uint32_t n, const uint32_t* faces_q, const float* bary, float* out);
/* MeshMap::meshAhead adds every layer's vectorAt to the planner's direction (mesh_map.cpp:1097-1102): enable != 0 makes
 * mnb_cvp_backtrack add the resident inflation field (config_.repulsive_field, inflation_layer.h:247). */
int32_t mnb_set_repulsive_field(mnb_ctx* ctx, int32_t enable);

/* ---- cancel (CVPMeshPlanner::cancel / DijkstraMeshPlanner::cancel) ------- */
int32_t mnb_cancel(mnb_ctx* ctx);

/* ---- introspection for tests / bench ------------------------------------ */
typedef struct mnb_stats {
  uint64_t rounds;          /* band rounds of the last wavefront call */
  uint64_t recomputes;      /* vertex recomputations (>= settled vertices) */
  uint64_t settled;         /* vertices with a finite final label */
  uint64_t kernel_launches; /* kernels launched by the last call */
  float kernel_ms;          /* CUDA-event time of the wavefront kernel(s) of the last call */
  uint64_t skipped;         /* candidate-rounds that kept their label without a recompute (clean-candidate skip) */
  uint64_t deep_labels;     /* mnb_cvp: labels whose pop time has more than 3 nested cascade levels (informational: the order is exact at any depth; their level stacks live in the per-wavefront level pool) */
  uint64_t pool_words;      /* words of the level pool used by the last wavefront call (max over concurrent wavefronts) */
} mnb_stats;
int32_t mnb_get_stats(mnb_ctx* ctx, mnb_stats* out);
/* tuning knobs: band width delta (metres) and CTAs per wavefront cluster (1,2,4,8,16) */
int32_t mnb_set_tuning(mnb_ctx* ctx, float band_delta, int32_t cluster_size, int32_t threads_per_cta);

/* ---- multi-GPU: one host process, N devices (SURVEY.md 8e; north star: "batched multi-goal queries shard one goal per
 * GPU ... with NCCL over NVLink only to gather the resulting potential arrays") ----------------------------------------
 * A group owns one mnb_ctx per device (mnb_group_ctx: use it for everything that is per device -- layers, single plans,
 * tuning) and the NCCL communicators of the gather.  NCCL is bound at run time (libnccl.so.2); a group of one device
 * never touches it.  Reference counterpart: none -- the reference plans one query per MBF action on one CPU thread
 * (mbf_mesh_nav/src/mesh_planner_execution.cpp:55-66); this is the batched form of CVPMeshPlanner::waveFrontPropagation
 * (cvp_mesh_planner.cpp:651-886) behind mnb_cvp_batch, sharded. */
typedef struct mnb_group mnb_group;
int32_t mnb_group_create(int32_t n_devices, const int32_t* devices /* CUDA ordinals */, mnb_group** out_group);
void mnb_group_destroy(mnb_group* group);
int32_t mnb_group_size(mnb_group* group);
mnb_ctx* mnb_group_ctx(mnb_group* group, int32_t rank);
const char* mnb_group_last_error(mnb_group* group);
/* replicate the map / the per-plan costs on every device (HOST pointers, as mnb_set_mesh / mnb_set_costs) */
int32_t mnb_group_set_mesh(mnb_group* group, uint32_t V, uint32_t F, const float* pos, const uint32_t* faces,
                           const uint32_t* edges, uint32_t E);
int32_t mnb_group_set_costs(mnb_group* group, const float* vertex_costs, const float* edge_weights, const uint8_t* invalid);
/* MeshMap::layerChanged (mnb_update_vertex_costs) on every replica of the group, all devices concurrently; HOST arrays */
int32_t mnb_group_update_vertex_costs(mnb_group* group, uint32_t n_changed, const uint32_t* changed, const float* costs,
                                      int32_t costs_indexed_by_vertex, float default_value, double edge_cost_factor);
/* n full-field plans, goal k on rank k mod N, all devices concurrently; with gather != 0 one in-place ncclAllGather leaves
 * every field on every device.  Result on each device: float[N][pad][V], pad = ceil(n / N), the field of goal k is row
 * mnb_group_row(group, k); the buffers belong to the group and stay valid until its next sharded call.  seed arrays: HOST.
 * Returns the MBF code / MNB_E_* of the first rank that failed. */
int32_t mnb_cvp_batch_sharded(mnb_group* group, uint32_t n, const uint32_t* seed_faces, const float* seed_pos /* 3n */,
                              double cost_limit, int32_t gather);
uint32_t mnb_group_row(mnb_group* group, uint32_t goal);
float* mnb_group_fields(mnb_group* group, int32_t rank /* device pointer on that rank's device */);
int32_t mnb_group_read_fields(mnb_group* group, int32_t rank, uint32_t first_goal, uint32_t count, float* out_host /* count*V */);

#ifdef __cplusplus
}
#endif
#endif /* MESHNAV_B200_H */
