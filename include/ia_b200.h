/*
 * ia_b200.h -- C ABI of libia_b200.so, the H100 (sm_90a) implementation of InstantAvatar's per-ray hot
 * path.  Plain pointers and sizes only; every pointer is a DEVICE pointer unless marked [host]; all
 * buffers are owned by the caller (the library never allocates, frees or retains pointers, and never
 * synchronises the device).  Every entry point enqueues work on `stream` and returns 0, or a negative
 * IA_E* code with a message retrievable through ia_last_error() (thread-local).
 *
 * Each entry point names the reference interface it replaces (paths relative to the reference repo
 * tijiang13/InstantAvatar @ 3cdfd49).
 */
#ifndef IA_B200_H
#define IA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define IA_ABI_VERSION 1
#define IA_NUM_INIT 13      /* deformers/fast_snarf/deformer_torch.py:28 */
#define IA_NUM_LEVELS 16    /* models/networks/ngp.py:30 */
#define IA_MLP_HALFS 22144  /* padded fp16 weight block (forward + transposed copies), see ia_params_to_half */
#define IA_ENC_MLP_PARAMS 3072
#define IA_COL_MLP_PARAMS 6144
#define IA_MAX_SAMPLES 256  /* confs/renderer/raymarcher_acc.yaml:2 */

#define IA_OK 0
#define IA_EINVAL (-1)
#define IA_ECUDA (-2)

typedef void* ia_stream_t; /* cudaStream_t */

/* Per-frame state of the nearest-vertex deformer (deformers/smpl_deformer.py:87-137, `deformer=smpl`): a sample x in the
 * root frame takes its nearest posed vertex v (squared fp32 distance dx*dx + dy*dy + dz*dz, ties to the lower index) and is
 * valid iff d2 < (float)(threshold * threshold); its canonical point is table[v] . [x, 1].  `grid` is a caller-owned
 * workspace of ia_nv_workspace_bytes(n_verts) bytes filled by ia_nv_grid_build from `verts`. */
typedef struct IaNearestVertex {
    void* grid;              /* vertex bucket grid (ia_nv_grid_build) */
    const float* verts;      /* [n_verts][3] posed vertices, root frame */
    const float* table;      /* [n_verts][12] rows 0..2 of T_inv[v] (3x4, row-major) */
    int32_t n_verts;
    double threshold;        /* smpl_deformer.py `threshold` (0.05) */
} IaNearestVertex;

/* Per-frame read-only state of the fused kernels. */
typedef struct IaScene {
    const float* field;      /* [D][H][W+1][12] fp32 written by ia_precompute: the blended 3x4 LBS transform (row-major) of each voxel
                              * once, rows padded with one zero voxel; the 24 floats from voxel x on are voxel x, then voxel x+1 */
    int32_t D, H, W;
    const float* offset_k;   /* [3] ForwardDeformer.offset_kernel (deformer_torch.py:154) */
    const float* scale_k;    /* [3] ForwardDeformer.scale_kernel  (deformer_torch.py:155-158) */
    const float* tfs;        /* [24][4][4] bone transforms (snarf_deformer.py:86) */
    const uint32_t* occ_bits;/* [G*G*G/32 + 8] occupancy bitfield, bit index (nx*G+ny)*G+nz (ia_pack_occupancy) */
    int32_t G;
    const float* occ_aabb;   /* [6] min xyz, max xyz of the occupancy grid (DensityGrid.min_corner/max_corner) */
    const void* table_h;     /* half2[total_entries] hash-grid features (ia_params_to_half) */
    const void* mlp_h;       /* half[IA_MLP_HALFS] padded MLP weights (ia_params_to_half) */
    const float* net_center; /* [3] NeRFNGPNet.center (ngp.py:64-71) */
    const float* net_scale;  /* [3] NeRFNGPNet.scale */
    /* [host] nullable.  Set: the deform stage is the nearest-vertex search instead of Fast-SNARF's root finding, and
     * field / offset_k / scale_k / tfs / D / H / W are not read.  Supported by ia_render_fwd, ia_occupancy_query,
     * ia_deform_query and ia_train_fwd_split; ia_render_fwd_peer, ia_occupancy_query_peer, ia_broyden and ia_pose_grad
     * return IA_EINVAL (the pose gradient is ia_nv_pose_grad). */
    const IaNearestVertex* nv;
} IaScene;

/* Work counters accumulated by the kernels (device memory, caller zeroes). */
typedef struct IaStats {
    unsigned long long samples;   /* occupied samples evaluated (M) */
    unsigned long long gathers;   /* trilinear field samples taken by Broyden (M*13*kbar) */
    unsigned long long net_evals; /* hash-grid + MLP evaluations (P) */
    unsigned long long rays_hit;  /* rays with at least one occupied sample */
    unsigned long long field_loads; /* of `gathers`, those that issued loads (4 x-pairs of 96 B each, counted as 12 sectors of 32 B): footprints outside the
                                     * skinning volume and early-out solves are exact zeros computed without memory traffic */
    unsigned long long hash_loads; /* hash-table loads issued per lane (one 32-byte sector each): 16 levels x 8 corners = 128 per
                                    * network evaluation */
} IaStats;

int ia_abi_version(void);
const char* ia_last_error(void);
/* number of SMs of the current device (grid sizing is a multiple of this) [host result] */
int ia_sm_count(void);

/* tuning knob (does not change results): "render_rays_per_warp" in {4, 2, 1} (ray tile of ia_render_fwd*; the sharded
 * frame uses 2 and 1).  Any other name is IA_EINVAL ("unknown option"). */
int ia_set_option(const char* name, int value);

/* tiny-cuda-nn HashGrid level table (models/networks/ngp.py:27-37 config). [host] outputs. */
int ia_hashgrid_layout(uint32_t res[IA_NUM_LEVELS], float scale[IA_NUM_LEVELS], uint32_t size[IA_NUM_LEVELS],
                       uint32_t offset[IA_NUM_LEVELS], uint32_t* total_entries);

/* Replaces precompute_cuda.precompute (deformers/fast_snarf/cuda/precompute/precompute.cpp:7-13,
 * precompute.cu:24-103).  voxel_w [24][D][H][W] skinning weights, tfs [24][4][4].
 * field_out [D][H][W+1][12]: D*H*(W+1)*12 floats, 16-byte aligned (a larger buffer works too), the row-major 3x4 of every voxel
 * and a zero voxel at the end of each row (IaScene.field); voxel_d_out [3][D][H][W] (nullable; reference layout, deformer.voxel_d);
 * aabb_out [6] = min/max of voxel_d (nullable; SNARFDeformer.get_bbox_deformed, snarf_deformer.py:105-107). */
int ia_precompute(const float* voxel_w, const float* tfs, const float* offset_k, const float* scale_k, int D, int H,
                  int W, float* field_out, float* voxel_d_out, float* aabb_out, ia_stream_t stream);

/* Once-per-subject voxelisation of the SMPL skinning weights (deformers/fast_snarf/deformer_torch.py:225-244
 * query_weights_smpl, called from switch_to_explicit :150-158): K nearest canonical vertices of every voxel centre
 * (pytorch3d knn_points contract: squared distances, ascending, ties keep the earlier vertex), weights
 * 1/clamp(sqrt(d2),1e-4,1) normalised, blended vertex skinning weights, then `smooth_passes` Jacobi passes
 * ((w-mean6)*0.7+mean6 on interior voxels, renormalise).  verts [n][3], vert_weights [n][24]; xs [W], ys [H], zs [D] =
 * torch.linspace(-1,1,.) grids; voxel centre = (xs[x], ys[y], zs[z]/ratio) * scale[0] + offset[3] (offset, scale:
 * device pointers, no host sync).  lbs_voxel [24][D][H][W] out; scratch same size (nullable if smooth_passes == 0). */
int ia_voxelize_weights(const float* verts, const float* vert_weights, int n_verts, const float* xs, const float* ys,
                        const float* zs, int D, int H, int W, const float* offset, const float* scale, float ratio,
                        int knn, int smooth_passes, float* lbs_voxel, float* scratch, ia_stream_t stream);

/* Nearest vertex of every point: SMPLDeformer.deform's ops.knn_points(pts, vertices, K=1)
 * (deformers/smpl_deformer.py:94-95; third_parties/pytorch3d/ops.py:123-206 contract: squared distance, ties keep the
 * earlier vertex).  pts [n][3], verts [n_verts][3] -> idx_out [n] int32, dist2_out [n]. */
int ia_knn1(const float* pts, int n, const float* verts, int n_verts, int* idx_out, float* dist2_out, ia_stream_t stream);

/* Nearest-vertex deformer, per frame: one CTA buckets nv->verts into a uniform grid in nv->grid (bounds, per-cell counts,
 * scan, scatter; cell edge >= 1.01 * threshold, widened if the cell count would exceed the workspace's capacity; the grid
 * is padded by one cell on every side).  No host synchronisation.  Every vertex within `threshold` of a point lies in the
 * 3x3x3 cells around it, so the search is exact for every valid point, and points outside the grid are invalid. */
size_t ia_nv_workspace_bytes(int n_verts);
int ia_nv_grid_build(const IaNearestVertex* nv /*[host]*/, ia_stream_t stream);
/* The grid search on its own (the grid analogue of ia_knn1): pts [n][3] -> idx_out [n] int32 and dist2_out [n] of the
 * nearest vertex for valid points (d2 < threshold^2; same index and bit-identical d2 as ia_knn1), -1 and +inf otherwise. */
int ia_nv_nearest(const IaNearestVertex* nv /*[host]*/, const float* pts, int n, int* idx_out, float* dist2_out,
                  ia_stream_t stream);

/* Per-frame bone transforms in one launch.  Replaces, for everything the renderer consumes, the SMPL forward + tfs
 * algebra of SNARFDeformer.prepare_deformer (deformers/snarf_deformer.py:79-86; smplx/lbs.py:295-329 Rodrigues,
 * :345-401 kinematic chain; body_models.py:353-360 transl): global_orient [3], body_pose [69], transl [3] (nullable),
 * joints [24][3] rest-pose joint locations of the subject (function of betas only; cached by the caller), parents [24]
 * (int32, -1 for the root), tfs_inv_t [24][4][4] inverse canonical-pose transforms (snarf_deformer.py:52).
 * Outputs tfs [24][4][4], w2s [4][4], A_out [24][4][4] (nullable). */
int ia_smpl_tfs(const float* global_orient, const float* body_pose, const float* transl, const float* joints,
                const int* parents, const float* tfs_inv_t, float* tfs, float* w2s, float* A_out, ia_stream_t stream);

/* Rays world -> SMPL-root frame, one launch.  Replaces SNARFDeformer.transform_rays_w2s
 * (deformers/snarf_deformer.py:95-103: two small GEMMs, a norm and two element-wise ops):
 *   o' = o R^T + t,  d' = d R^T   with [R | t] = w2s[:3, :4],   near = |o'| - 1,   far = |o'| + 1.
 * rays_o / rays_d [.][3] (inputs), w2s [4][4] row-major (device); outputs o_out / d_out [n][3], near_out / far_out [n].
 * index (int32 [n], nullable): output ray i is input ray index[i] -- a rank of a ray-sharded frame picks its tiles in the
 * same launch.  Without index, in-place use (o_out == rays_o, d_out == rays_d) is allowed. */
int ia_transform_rays(const float* w2s, const float* rays_o, const float* rays_d, const int* index /*nullable*/, int n,
                      float* o_out, float* d_out, float* near_out, float* far_out, ia_stream_t stream);

/* Reverse mode of ia_smpl_tfs for pose optimisation (what autograd computes through smplx/lbs.py:295-329,345-401 and
 * snarf_deformer.py:84-86): grad_tfs [24][4][4] -> grad_orient [3] (nullable), grad_pose [69], grad_transl [3]
 * (nullable).  Values are written, not accumulated.  tfs is relative to the root, so grad_orient / grad_transl come out
 * as the fp32 residue of an exact cancellation -- as they do in the reference. */
int ia_smpl_tfs_backward(const float* global_orient, const float* body_pose, const float* transl, const float* joints,
                         const int* parents, const float* tfs_inv_t, const float* grad_tfs, float* grad_orient,
                         float* grad_pose, float* grad_transl, ia_stream_t stream);

/* fp32 master parameters -> fp16 working copies (tiny-cuda-nn casts params to fp16 every forward).
 * enc_params [3072 + 2*total] = [W1 64x32 | W2 16x64 | grid]; col_params [6144] = [W3 64x16 | W4 64x64 | W5 16x64]
 * (models/networks/ngp.py:27-57 `encoder.params`, `color_net.params`). */
int ia_params_to_half(const float* enc_params, const float* col_params, void* table_h, void* mlp_h,
                      ia_stream_t stream);

/* bool [G][G][G] (DensityGrid.density_field) -> bitfield.  bits must hold G*G*G/32 + 8 words: the 8 trailing
 * words receive the bounding box of the occupied cells (used for exact empty-space skipping). */
int ia_pack_occupancy(const uint8_t* field_bool, uint32_t* bits, int G, ia_stream_t stream);

/* Occupancy-grid post-processing on the device: density [G][G][G] (already EMA'd / max-merged by the caller) ->
 * 1-exp(-0.01 d), 3x3x3 max-pool, > min(mean, 0.01), largest 26-connected component.  Replaces
 * models/structures/density_grid.py:78-85 / :104-110 incl. max_connected_component (:118-125).
 * field_out bool [G][G][G] (nullable), bits_out [G*G*G/32 + 8]; workspace >= 12*G^3 + 64 bytes. */
int ia_occupancy_build(const float* density, int G, uint8_t* field_out, uint32_t* bits_out, void* workspace,
                       size_t workspace_bytes, ia_stream_t stream);

/* demo.yaml's `smpl_init` (DESIGN.md §3.6, §5.13): the first step-< 500 grid update of a training frame seeds its grid
 * from the posed SMPL mesh (density_grid.py:52-68, kaolin's point_to_mesh_distance and check_sign).
 *
 * ia_smpl_init_seed: unless *seeded != 0 (then the field and cache are left as they are), over the cell centres
 *   c_i = (i / G + 0.5 / G) * ext + lo (float32, per axis; lo, ext from aabb6 = min xyz, max xyz) of a G^3 grid
 *   (x slowest): field_out[c] = sqrtf(d2) < 0.01f || inside(c), with d2 the float32 squared distance to the nearest of
 *   the n_faces triangles faces [n_faces][3] (int32 indices into verts [n_verts][3], each in [0, n_verts): the caller
 *   guarantees it, the kernels do not check) and inside(c) the parity of the
 *   crossings of the +z ray from c with the triangles (a triangle covers a column when the three edge functions of its
 *   xy projection, each evaluated in the canonical order of its endpoints, share one sign; a zero edge function takes
 *   the sign at the point moved by (eps, eps^2)); cache[c] = max(0.8 cache[c], field ? +inf : 0).  Then bits_out
 *   [G^3/32 + 8] = ia_pack_occupancy(field_out) (unchanged for a seeded frame) and *seeded = 1.  seeded: device int32 [1].
 *   workspace: device, ia_smpl_init_workspace_bytes(G) bytes.  No host synchronisation.
 *   IA_EINVAL: G not a multiple of 32 in [32, 1024], n_verts < 1, n_faces < 0, a short workspace, a NULL pointer.
 * ia_occupancy_frame_copy: f = clamp(*idx, 0, n_frames - 1) (idx: device int64 [1]); store = 0 copies frame f of the
 *   stacked grids (cache_all [n_frames][G^3] fp32, field_all [n_frames][G^3] bool, bits_all [n_frames][G^3/32 + 8],
 *   seeded_all [n_frames] int32) into the working grid (cache, field, bits, seeded [1]); store = 1 copies it back.
 *   cache_all, field_all, cache and field 16-byte aligned.  IA_EINVAL: n_frames < 1, a bad G or store, a NULL pointer,
 *   a misaligned pointer. */
size_t ia_smpl_init_workspace_bytes(int G);
int ia_smpl_init_seed(const float* verts, int n_verts, const int* faces, int n_faces, const float* aabb6, int G,
                      int32_t* seeded, float* cache, uint8_t* field_out, uint32_t* bits_out, void* workspace,
                      size_t workspace_bytes, ia_stream_t stream);
int ia_occupancy_frame_copy(const int64_t* idx, int n_frames, int G, float* cache_all, uint8_t* field_all, uint32_t* bits_all,
                            int32_t* seeded_all, float* cache, uint8_t* field, uint32_t* bits, int32_t* seeded, int store,
                            ia_stream_t stream);

/* Marching cubes (replaces skimage.measure.marching_cubes in utils/marching_cubes.py:29-30 and trimesh's
 * matrix_to_marching_cubes in DensityGrid.export_mesh, density_grid.py:112-116).  field [nx][ny][nz] fp32, x slowest;
 * nx, ny, nz >= 2 and 3*nx*ny*nz < 2^31, else IA_EINVAL (and the *_bytes queries return 0).  A lattice point is above
 * iff v > level; every lattice edge with exactly one end above carries one vertex, id ordered by (linear index of the
 * lower end, axis).  Triangles come from the generated table ia_mc_table.cuh, ordered by (cube linear index, table
 * order).  Two calls share the caller's workspace of ia_mc_workspace_bytes(nx, ny, nz) bytes:
 *   ia_mc_count : counts [3] int64 (device) = {n_verts, n_faces, number of non-finite field values}
 *   ia_mc_emit  : verts [n_verts][3] = (p / div) * ext + origin per component (p: index-space position, the crossing
 *                 axis at i + (level - v_lo) / (v_hi - v_lo); ext_origin [6] device = ext xyz, origin xyz), faces
 *                 [n_faces][3] int32; flip = 0: triangle normals point to the above side (object {v < level}),
 *                 flip != 0: to the other side.  n_verts / n_faces: the counts of ia_mc_count. */
size_t ia_mc_workspace_bytes(int nx, int ny, int nz);
int ia_mc_count(const float* field, int nx, int ny, int nz, float level, void* workspace, size_t workspace_bytes,
                long long* counts, ia_stream_t stream);
int ia_mc_emit(const float* field, int nx, int ny, int nz, float level, int flip, float div, const float* ext_origin,
               const void* workspace, size_t workspace_bytes, int n_verts, int n_faces, float* verts, int* faces,
               ia_stream_t stream);

/* Largest connected component of a triangle mesh (trimesh.Trimesh.split + the max-area choice of
 * utils/marching_cubes.py:36-45 + submesh): faces sharing a vertex are connected; a component's area is the exact sum
 * of its faces' float32 0.5 |(b - a) x (c - a)| in 2^-32 fixed point (exact while below 2^32 units^2); the largest area
 * wins, an exact tie goes to the component holding the lowest face index.  The kept faces keep their order, the kept
 * vertices their ascending order, re-indexed: verts_out [n_verts][3] and faces_out [n_faces][3] (capacity) receive
 * kept [2] int64 (device) = {vertices, faces} rows.  workspace >= ia_mc_component_workspace_bytes(n_verts, n_faces). */
size_t ia_mc_component_workspace_bytes(int n_verts, int n_faces);
int ia_mc_largest_component(const float* verts, const int* faces, int n_verts, int n_faces, void* workspace,
                            size_t workspace_bytes, float* verts_out, int* faces_out, long long* kept,
                            ia_stream_t stream);

/* Fused eval renderer.  Replaces Raymarcher.render_test (renderers/raymarcher_acc.py:82-138) together with
 * raymarch_test / composite_test (renderers/cuda/raymarcher.cpp:16-29,65-75), SNARFDeformer.deform_test
 * (deformers/snarf_deformer.py:126-141), fuse_broyden + filter (fuse_cuda.cpp:14-25, filter.cpp:12-18) and
 * NeRFNGPNet.forward (models/networks/ngp.py:73-83).
 * rays_o/rays_d [n][3], near/far [n] in the SMPL-root frame (after transform_rays_w2s); bg [n][3] or NULL (white).
 * Outputs rgb [n][3], depth [n], alpha [n], counter [n] (occupied samples evaluated per ray).
 * image_width: optional hint (>0: rays are a row-major image of that width -> small pixel tiles per warp).
 * workspace: >= 256 bytes; with >= ia_render_workspace_bytes(n_rays) the tiles are scheduled longest-first from a
 * cheap planning pass (same results).  stats: nullable. */
size_t ia_render_workspace_bytes(int n_rays);
int ia_render_fwd(const IaScene* scene /*[host]*/, const float* rays_o, const float* rays_d, const float* near,
                  const float* far, int n_rays, const float* bg, int image_width, float* rgb, float* depth,
                  float* alpha, float* counter, void* workspace, size_t workspace_bytes, IaStats* stats,
                  ia_stream_t stream);

/* Ray-sharded frame over peer memory (one process per GPU, NVLink): as ia_render_fwd, and additionally the RGBA of ray i
 * is stored straight into the [n_pixels][4] fp32 image of every peer at pixel pixel_index[i] (int32 [n_rays]; NULL: i).
 * peer_rgba: DEVICE array of n_peers image pointers (symmetric-memory mappings of the peers' buffers).  The caller
 * separates frames with a cross-GPU barrier; no gather collective is needed.  (No counterpart in the reference, which is
 * single-GPU: BASELINE.json config 3.) */
int ia_render_fwd_peer(const IaScene* scene /*[host]*/, const float* rays_o, const float* rays_d, const float* near,
                       const float* far, int n_rays, const float* bg, int image_width, float* rgb, float* depth,
                       float* alpha, float* counter, void* workspace, size_t workspace_bytes, IaStats* stats,
                       const int* pixel_index, float* const* peer_rgba, int n_peers, ia_stream_t stream);

/* Point query: per point, max density over the valid canonical correspondences.  Replaces
 * SNARFDeformer.__call__(pts, model, eval_mode) (deformers/snarf_deformer.py:126-165), used by
 * DensityGrid.update / initialize (models/structures/density_grid.py:46-110).
 * pts [n][3]; eval_mode != 0: invalid sigma = 0 and nan_to_num, else invalid sigma = -1e5.
 * Outputs rgb [n][3], sigma [n]; xc_best [n][3] (nullable; canonical point of the arg-max candidate, 0 if none);
 * best_init [n] int8 (nullable; index 0..12 of the winning initialisation, -1 if none valid). */
int ia_deform_query(const IaScene* scene /*[host]*/, const float* pts, int n, int eval_mode, float* rgb, float* sigma,
                    float* xc_best, int8_t* best_init, IaStats* stats, ia_stream_t stream);

/* DensityGrid.initialize's density pass (models/structures/density_grid.py:94-103): for each of `passes` jitter tensors
 * [G][G][G][3] the G^3 cell points (idx/G + jitter/G) * (max - min) + min are queried in eval mode and max(sigma, 0) is
 * reduced into density_max [G][G][G] (zeroed by the library).  aabb [6] device.  Two launches: root finding appends every
 * kept root to a list in `workspace`, then the network evaluates the list.  workspace: device, at least
 * ia_occupancy_query_workspace_bytes(G, passes, n_shards) bytes.  shard / n_shards: this call evaluates every n_shards-th
 * batch of cells starting at `shard` (multi-GPU: the caller max-all-reduces density_max; 0 / 1 = all). */
int ia_occupancy_query(const IaScene* scene /*[host]*/, const float* jitter, const float* aabb, int G, int passes,
                       float* density_max, void* workspace, int shard, int n_shards, IaStats* stats, ia_stream_t stream);
/* bytes of ia_occupancy_query*'s workspace: counters, root-finding scratch and a root list that holds the shard's worst
 * case (all 13 roots of every grid point kept; 272 MB at G = 64, 5 passes, 1 shard); 0 for invalid arguments [host] */
size_t ia_occupancy_query_workspace_bytes(int G, int passes, int n_shards);

/* ia_occupancy_query over peer memory: this rank's shard of the cells is max-reduced into the density grid of EVERY rank
 * with NVLink atomics (positive densities only: ~2 % of the cells), replacing the 1 MB max-all-reduce.  peer_density: DEVICE
 * array of n_peers pointers to [G][G][G] fp32 buffers, zeroed by their owners before the barrier that precedes the launch. */
int ia_occupancy_query_peer(const IaScene* scene /*[host]*/, const float* jitter, const float* aabb, int G, int passes,
                            float* const* peer_density, int n_peers, void* workspace, int shard, int n_shards,
                            IaStats* stats, ia_stream_t stream);

/* Measurement aid (bench.py `roofline.peak`): the fused kernels' memory access shape in isolation -- every lane gathers
 * trilinear footprints (4 x-pairs of 96 B = 24 LDG.128, 3-4 32-byte sectors per pair) from the L2-resident field `field`
 * (IaScene.field layout), the next footprint depending on the loaded data -- at one persistent CTA of `warps` (12 / 16 / 24 / 32)
 * warps per SM.  coherent != 0: the lanes of a warp stay within a 10 x 3 x 3 voxel neighbourhood (a batch of the
 * occupancy query).  *sectors_out (device) += 12 sectors per footprint (nominal, 3 per pair); the caller times the launch with CUDA events. */
int ia_gather_ceiling(const float* field, int D, int H, int W, int iters, int warps, int coherent,
                      unsigned long long* sectors_out, float* sink /*nullable*/, ia_stream_t stream);

/* Fine-grained entry points (serve the legacy `model(pts)` callback path and the tinycudann-named shim):
 * ia_broyden replaces fuse_kernel.fuse_broyden + filter_cuda.filter
 *   (deformer_torch.py:100-116): xd [n][3] -> xc [n][13][3] (0 where invalid), valid [n][13] (after filter),
 *   j_inv [n][13][9] (nullable).
 * ia_ngp_forward replaces NeRFNGPNet.forward: x [n][3] canonical points -> sigma [n], rgb [n][3]. */
int ia_broyden(const IaScene* scene /*[host]*/, const float* xd, int n, float* xc, uint8_t* valid, float* j_inv,
               ia_stream_t stream);
int ia_ngp_forward(const IaScene* scene /*[host]*/, const float* x, int n, float* sigma, float* rgb,
                   ia_stream_t stream);

/* The two tiny-cuda-nn modules of models/networks/ngp.py:27-57 as separate operators -- what the in-repo `tinycudann`
 * module (tcnn.NetworkWithInputEncoding / tcnn.Network with flat fp32 `params`, fp16 outputs, internal loss scale) binds, so
 * that the reference's ngp.py runs verbatim on these kernels:
 *   ia_tcnn_encoder_forward : x01 [n][3] in [0,1] -> out16 [n][16] fp16 (HashGrid 16 x 2, 2^19, base 16, scale 1.5 +
 *                             FullyFusedMLP 32 -> 64 ReLU -> 16); scene needs table_h and mlp_h
 *   ia_tcnn_encoder_backward: d loss / d out16 [n][16] fp32 -> grad_enc [3072 + 2*total] (+=; nullable) and/or denc_out
 *                             [n][32] (d loss / d hash features, for the input gradient via ia_ngp_input_grad)
 *   ia_tcnn_mlp_forward     : in15 [n][15] fp32 -> out3 [n][3] fp16 (15 (+1.0 pad) -> 64 -> 64 -> 3, ReLU, sigmoid output)
 *   ia_tcnn_mlp_backward    : d loss / d out3 [n][3] fp32 -> grad_col [6144] (+=; nullable) and/or din15 [n][15]
 * scratch >= ia_tcnn_backward_scratch_bytes(n); grad_*_dummy: 6144 / 3072 floats the shared weight-gradient pass may touch
 * (the other module's all-zero contribution).  mlp_h as produced by ia_mlp_to_half. */
size_t ia_tcnn_backward_scratch_bytes(int n);
int ia_tcnn_encoder_forward(const IaScene* scene /*[host]*/, const float* x01, int n, void* out16_h, ia_stream_t stream);
int ia_tcnn_encoder_backward(const IaScene* scene /*[host]*/, const float* x01, const float* dout16, int n, float grad_scale,
                             float* grad_enc, float* grad_col_dummy, void* scratch, float* denc_out, ia_stream_t stream);
int ia_tcnn_mlp_forward(const void* mlp_h, const float* in15, int n, void* out3_h, ia_stream_t stream);
int ia_tcnn_mlp_backward(const void* mlp_h, const float* in15, const float* dout3, int n, float grad_scale, float* grad_col,
                         float* grad_enc_dummy, void* scratch, float* din15, ia_stream_t stream);

/* Kernel-for-kernel replacements of the reference's raymarcher extension (renderers/cuda/raymarcher.cpp:16-81), for
 * the legacy `model(pts)` callback path.  Layouts are the reference's: density_grid bool [G][G][G], alive int64,
 * outputs zero-initialised by the caller (the reference allocates them with at::zeros), `nears` / `color` / `depth` /
 * `no_hit` updated in place. */
int ia_raymarch_train(const float* rays_o, const float* rays_d, const float* nears, const float* fars, int n_rays,
                      const uint8_t* density_grid, int grid_size, const float* scale, const float* offset,
                      const float* step_size, int N_steps, float* depths, ia_stream_t stream);
int ia_raymarch_test(const float* rays_o, const float* rays_d, float* nears, const float* fars, const int64_t* alive,
                     int n_alive, const uint8_t* density_grid, int grid_size, const float* scale, const float* offset,
                     const float* step_size, int N_steps, float* pts, float* deltas, float* depths, ia_stream_t stream);
int ia_composite_test(const float* rgb_vals, const float* sigma_vals, const float* delta_vals, const float* depth_vals,
                      const int64_t* alive, int n_alive, int N_steps, float* color, float* depth, float* no_hit,
                      float thresh, ia_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------
 * Training path
 * --------------------------------------------------------------------------------------------------------- */

/* Training forward.  Replaces Raymarcher.render_train (renderers/raymarcher_acc.py:140-186) together with
 * raymarch_train (raymarcher.cpp:41-53), SNARFDeformer.deform_train (snarf_deformer.py:143-159) and the network, in
 * three launches: (1) march -- one warp per ray, at most 1024 steps, occupied steps become consecutive slots, their
 * jittered posed points are appended to a device-side sample list, except those of slots whose un-jittered depth is
 * <= 0 (near <= 0), which keep s_rgb 0, s_sigma -1e3 and s_best -1 as in :156-162; (2) the point-query kernel over that list, every 32-sample batch an
 * independent work item of all resident warps; (3) per-ray compositing.  Its time scales with the number of samples.
 * jitter [n][256] (U(0,1), replaces torch.rand_like, :158) and noise [n][256] (already scaled, replaces
 * noise*randn_like, :167) are nullable.  Outputs rgb [n][3], depth [n], alpha [n], weights [n][256] and the dense
 * per-sample state the backward needs: s_sigma/s_z [n][256], s_rgb/s_xc [n][256][3], s_best [n][256] (int8, -1 =
 * no valid root), s_count [n]; past s_count, weights are 0, s_best is -1 and the other slots are unspecified.  workspace:
 * ia_train_fwd_workspace_bytes(n_rays) (256 + 4 * n_rays * 256). */
size_t ia_train_fwd_workspace_bytes(int n_rays);
int ia_train_fwd_split(const IaScene* scene /*[host]*/, const float* rays_o, const float* rays_d, const float* near,
                       const float* far, int n_rays, const float* bg, const float* jitter, const float* noise, float* rgb,
                       float* depth, float* alpha, float* weights, float* s_sigma, float* s_rgb, float* s_xc, float* s_z,
                       int* s_count, int8_t* s_best, void* workspace, size_t workspace_bytes, IaStats* stats,
                       ia_stream_t stream);

/* Compositing backward (autograd of raymarcher_acc.py:25-36,166-186): upstream grads (nullable) of rgb [n][3],
 * depth [n], alpha [n], weights [n][256] -> compact list of (canonical point, d sigma, d rgb) of the samples that
 * reached the network; l_* arrays hold up to n*256 entries, l_count [1] must be zeroed by the caller. */
int ia_composite_bwd(int n_rays, const float* near, const float* far, const float* bg, const float* noise,
                     const float* s_sigma, const float* s_rgb, const float* s_xc, const float* s_z, const int* s_count,
                     const int8_t* s_best, const float* g_rgb, const float* g_depth, const float* g_alpha,
                     const float* g_weights, float* l_xc, float* l_dsigma, float* l_drgb, int* l_count,
                     const float* rays_o /*nullable*/, const float* rays_d /*nullable*/, float* l_xd /*nullable [n*256][3]*/,
                     int8_t* l_best /*nullable [n*256]*/, ia_stream_t stream);

/* Network backward (tiny-cuda-nn's autograd through HashGrid + FullyFusedMLPs, ngp.py:73-83): for the first
 * min(*count, capacity) list entries accumulates (+=) d loss / d encoder.params into grad_enc [3072 + 2*total] and
 * d loss / d color_net.params into grad_col [6144] (fp32, tcnn parameter order).  grad_scale: internal loss scale of
 * the fp16 dgrad chain (results are un-scaled).  scratch >= ia_ngp_backward_scratch_bytes(capacity). */
size_t ia_ngp_backward_scratch_bytes(int capacity);
int ia_ngp_backward(const IaScene* scene /*[host]*/, const float* xc, const float* dsigma, const float* drgb,
                    const int* count, int capacity, float grad_scale, float* grad_enc, float* grad_col, void* scratch,
                    float* denc_out /*nullable [capacity][32]: d loss / d hash features, input of ia_pose_grad;
                                      grad_enc and grad_col may both be null (frozen network) when denc_out is given*/,
                    ia_stream_t stream);

/* d loss / d x [n][3] of NeRFNGPNet.forward's input (tiny-cuda-nn's input gradient of HashGrid through the bbox
 * normalisation of ngp.py:75-77) from denc [n][32] = d loss / d (hash features) as written by ia_ngp_backward. */
int ia_ngp_input_grad(const IaScene* scene /*[host]*/, const float* x, const float* denc, int n, float* dx, ia_stream_t stream);

/* Pose gradients (SNARF_NGP_refine / optimize_SMPL): d loss / d tfs [24][4][4] (+=) through Fast-SNARF's implicit
 * differentiation (deformers/fast_snarf/deformer_torch.py:50-67, version 1): for each list sample the winning
 * initialisation's Broyden solve is re-run from xd (posed point) to recover x_c and the J_inv the reference stores, the
 * network's input gradient is formed from denc (ia_ngp_backward) and the hash-grid interpolation weights, and
 * -J_inv^T g (x) [x_c,1] is accumulated per bone with the border-padded trilinear skinning weights of
 * lbs_voxel [24][D][H][W] (ForwardDeformer.lbs_voxel_final). */
int ia_pose_grad(const IaScene* scene /*[host]*/, const float* lbs_voxel, const float* xd, const int8_t* best,
                 const float* denc, const int* count, int capacity, float* grad_tfs, ia_stream_t stream);

/* Forward linear-blend skinning of points into n_frames poses in one launch (ForwardDeformer.forward_skinning /
 * query_weights / skinning_mask, deformers/fast_snarf/deformer_torch.py:118-128,190-218).  Each point's 24 weights are
 * sampled once from lbs_voxel [24][D][H][W] (ForwardDeformer.lbs_voxel_final; trilinear, align_corners, border padding) at
 * scale_k * (x_c + offset_k) (offset_k, scale_k [3] as in IaScene), in the summation order of ia_pose_grad; then per frame
 * T = sum_j w_j tfs[f][j] and x_d = T[:3,:4] [x_c, 1] (DESIGN.md §3, "Forward skinning").  tfs [n_frames][24][4][4],
 * xc [n][3] -> xd [n_frames][n][3], weights [n][24] (nullable).  n = 0: nothing is done; n_frames < 1, n < 0 or
 * D / H / W < 1: IA_EINVAL. */
int ia_skin_points(const float* lbs_voxel, int D, int H, int W, const float* offset_k, const float* scale_k,
                   const float* tfs, int n_frames, const float* xc, int n, float* xd, float* weights /*nullable*/,
                   ia_stream_t stream);

/* Per-vertex skinning weights for a rig (DESIGN.md §3, "Rigged export").  Each vertex of xc [n][3] samples its 24 weights
 * exactly as ia_skin_points does, keeps the K largest in descending order (a tie goes to the lower joint index) and
 * divides them by their sum, accumulated in stored order: joints [n][K] uint8, weights [n][K].  A kept weight of exactly 0
 * is stored as joint 0, weight 0.  dropped [n] (nullable) receives the sum of the 24 - K weights not kept, in joint order.
 * A vertex whose kept sum is not positive gets joint 0 with weight 1 (then zeros) and adds 1 to *n_fallback (device int,
 * accumulated).  n = 0: nothing is done; K not in {4, 8, ..., 24}, n < 0 or D / H / W < 1: IA_EINVAL. */
int ia_vertex_skin_weights(const float* lbs_voxel, int D, int H, int W, const float* offset_k, const float* scale_k,
                           const float* xc, int n, int K, uint8_t* joints, float* weights, float* dropped /*nullable*/,
                           int* n_fallback, ia_stream_t stream);

/* Texture baking (DESIGN.md §3, "Texture baking"; the layout is csrc/ia_atlas.cuh's).  An atlas of size x size texels
 * (x right, y down, row 0 on top) gives faces 2k and 2k+1 the square cell k of c = floor(size / n) texels, n =
 * ceil(sqrt(ceil(n_faces / 2))) cells per row, at origin ((k mod n) c, (k div n) c); with L = c - 5, face 2k's corners
 * are (1, 1), (1 + L, 1), (1, 1 + L) and face 2k+1's (c - 1, c - 1), (c - 1 - L, c - 1), (c - 1, c - 1 - L) in the cell.
 * A texel belongs to face f when its centre lies within L-infinity distance 1 of f's triangle (at most one owner; all
 * four bilinear taps of a point of the triangle are f's).
 * ia_texture_atlas: layout = (n, c, L) of n_faces faces at `size`.  Host only, no GPU needed.
 * ia_texture_points: over all texels (t = row * size + column): owner [size^2] int32 = the owning face or -1, points
 *   [size^2][3] = b0 v0 + b1 v1 + b2 v2 in float32 for the barycentrics of the point of the face's flat triangle closest
 *   (Euclidean, in texel space) to the texel centre (the centre itself inside the triangle; not moved onto any level set),
 *   v_k = verts[faces[f][k]], and 0 for an unowned texel; uv [n_faces][3][2] (nullable) = the corners / size, glTF's
 *   TEXCOORD_0 (OBJ's vt flips v: 1 - y / size).  faces [n_faces][3] int32 indices into verts [n_verts][3]: each in
 *   [0, n_verts), the caller guarantees it (the kernel does not check).  n_faces = 0: nothing is done.
 * Both: IA_EINVAL for size outside [64, 16384], n_faces < 0 (< 1 for ia_texture_atlas), c < 6 (the message names the
 *   smallest size that fits) or a NULL pointer. */
int ia_texture_atlas(int n_faces, int size, int layout[3]);
int ia_texture_points(const float* verts, int n_verts, const int* faces, int n_faces, int size, int* owner, float* points,
                      float* uv /*nullable*/, ia_stream_t stream);

/* Pose gradient of the nearest-vertex deformer (scene->nv set).  For each of the first min(*count, capacity) list samples
 * of ia_composite_bwd with best >= 0: l_rz [capacity][3] holds (ray index, z, 0) -- what ia_composite_bwd writes into l_xd
 * when it is given the rays rays_o[i] = (i, 0, 0), rays_d[i] = (0, 1, 0) (z * 0 + i and z * 1 + 0 are exact).  The posed
 * point x = z * rays_d[ray] + rays_o[ray] is recomputed as the forward generated it, the forward's nearest-vertex search is
 * re-run from it (bit-identical), g = d loss / d x_c is formed from denc (ia_ngp_backward) as ia_ngp_input_grad does, and
 * accumulated (+=): grad_table [n_verts][3][4] += g (x) [x, 1] (d loss / d nv->table); grad_rays_o [n_rays][3] += T^T g and
 * grad_rays_d [n_rays][3] += z T^T g with T = table[v][:3][:3] (both nullable: d loss / d rays through x = z d + o). */
int ia_nv_pose_grad(const IaScene* scene /*[host]*/, const float* rays_o, const float* rays_d, int n_rays, const float* l_rz,
                    const int8_t* best, const float* denc, const int* count, int capacity, float* grad_table,
                    float* grad_rays_o /*nullable*/, float* grad_rays_d /*nullable*/, ia_stream_t stream);

/* NeRFLoss forward + analytic backward in one pass (instant_avatar/utils/loss.py:53-79):
 * loss = w_rgb mse(rgb) + w_alpha mse(alpha) + w_reg (mean reg(alpha) + mean reg(weights) + 2*0.313262),
 * reg(x) = -log(exp(-x) + exp(x-1)).  sums [12] (zeroed by the library): [0..3] = {sum (rgb-t)^2, sum (alpha-a)^2,
 * sum reg(alpha), sum reg(w)}, [4..8] = {mse_loss, loss_alpha_coarse, reg_alpha, reg_density, loss} as the reference logs
 * them (written by the last block to finish: no element-wise launches follow), [11] = block ticket.
 * g_* receive d loss / d output times *scale_dev (GradScaler scale; NULL = 1). */
int ia_nerf_loss(int n_rays, int n_samples, const float* rgb, const float* alpha, const float* weights,
                 const float* target_rgb, const float* target_alpha, float w_rgb, float w_alpha, float w_reg,
                 const float* scale_dev, float* g_rgb, float* g_alpha, float* g_weights, float* sums, ia_stream_t stream);

/* NGPLoss forward + analytic backward (instant_avatar/utils/loss.py:8-51) on patch-major rays: patch p holds rays
 * [p * patch_rays, (p + 1) * patch_rays) ([B, P, h, w] flattened, patch_rays = h * w; n_rays % patch_rays != 0 ->
 * IA_EINVAL).  NeRFLoss's terms give the same per-element gradients as ia_nerf_loss, bit for bit.  Added:
 *   depth-variance regulariser  L_d = (1/N) sum_i a_i |d_i - mu_p|,  mu_p = sum_p d a / S_p,  S_p = sum_p a + 1e-3,
 *   N = n_rays, weighted by w_depth_reg; with s_i = sign(d_i - mu_p) (0 at equality) and K_p = sum_p a s:
 *   dL_d/dd_i = (a_i s_i - K_p a_i / S_p) / N,  dL_d/da_i = (|d_i - mu_p| - K_p (d_i - mu_p) / S_p) / N.
 *   Each patch is reduced by one CTA in a fixed order: g_depth and g_alpha are the same in every run.
 *   g_rgb_extra [n_rays][3] (nullable): a further d loss / d rgb (the LPIPS term, evaluated by the caller), added to g_rgb.
 * All gradients are multiplied by *scale_dev (NULL = 1).  g_depth is written (zero when w_depth_reg == 0).
 * sums [16] (zeroed by the library): ia_nerf_loss's layout ([0..3] sums, [4..8] terms, [8] = NeRFLoss total, [11] block
 * ticket) plus [9] = sum a |d - mu|, [10] = loss_depth_reg, [12] = NeRFLoss total + w_depth_reg * loss_depth_reg. */
int ia_ngp_loss(int n_rays, int n_samples, int patch_rays, const float* rgb, const float* alpha, const float* depth,
                const float* weights, const float* target_rgb, const float* target_alpha, float w_rgb, float w_alpha,
                float w_reg, float w_depth_reg, const float* g_rgb_extra /*nullable*/, const float* scale_dev /*nullable*/,
                float* g_rgb, float* g_alpha, float* g_depth, float* g_weights, float* sums, ia_stream_t stream);

/* Fused dense Adam (torch.optim.Adam semantics, models/DNeRF.py:46-50) on a flat fp32 tensor; gradients are
 * multiplied by inv_grad_scale (GradScaler unscale, DNeRF.py:157-158); if found_inf (device, nullable) is non-zero
 * the step is skipped.  ia_grad_check_finite sets *found_inf = 1 when any gradient is non-finite. */
int ia_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, long n, float lr, float beta1,
                 float beta2, float eps, int step, float inv_grad_scale, const float* grad_scale_dev /*nullable: divides*/,
                 const float* found_inf, ia_stream_t stream);
int ia_grad_check_finite(const float* grads, long n, float* found_inf, ia_stream_t stream);

/* CUDA-graph friendly variant: every per-step scalar lives in device memory.  state [8] floats =
 * {lr, beta1, beta2, eps, step, bc1, bc2_sqrt, inv_scale}.  ia_adam_prepare (one thread) increments state[4] unless
 * *found_inf, recomputes the bias corrections and inv_scale = inv_world / *grad_scale_dev (1 if NULL).
 * ia_adam_step_dev applies the update (skipped when *found_inf), ALWAYS zeroes the gradient it consumed, and, when
 * half_out is non-NULL, refreshes the fp16 working copy half_out[i - half_skip] = half(params[i]) for i >= half_skip. */
int ia_adam_prepare(float* state, float inv_world, const float* grad_scale_dev, const float* found_inf, ia_stream_t stream);
int ia_adam_step_dev(float* params, float* grads, float* exp_avg, float* exp_avg_sq, long n, const float* state,
                     const float* found_inf, void* half_out, long half_skip, ia_stream_t stream);
/* Sharded optimiser over NVLink peer memory (one process per GPU; every rank's flat gradient, flat fp16 image and a
 * G-float flag array mapped into every peer, e.g. torch symmetric memory).  Replaces ncclReduceScatter + finite check +
 * Adam + ncclAllGather of the NCCL path by two kernels with the exchanges inside:
 *   ia_peer_reduce_check : shard_sum[i] = sum_r peer_grads[r][shard_off + i] (rank order; read through the peer
 *                          mappings), tested for non-finite values; on a hit (or *found_in != 0) flag[rank] = 1 is stored
 *                          into EVERY rank's flag array.                          -- cross-GPU barrier --
 *   ia_peer_flags_to_found: *found_inf = OR of this rank's flag array; flags reset.
 *   ia_adam_step_dev_peer: ia_adam_step_dev on the shard (grads = shard_sum) whose fp16 image is stored into EVERY rank's
 *                          flat image at element shard_off + i.                   -- cross-GPU barrier --
 * peer_grads / peer_flags / peer_half: DEVICE arrays of n_peers pointers.  The caller zeroes its gradient buffer after the
 * first barrier (all peers have read it). */
int ia_peer_reduce_check(const float* const* peer_grads, int n_peers, long shard_off, long shard_elems, float* shard_sum,
                         float* const* peer_flags, int rank, const float* found_in /*nullable*/, ia_stream_t stream);
int ia_peer_flags_to_found(float* flags, int n_peers, float* found_inf, ia_stream_t stream);
int ia_adam_step_dev_peer(float* params, float* grads, float* exp_avg, float* exp_avg_sq, long n, const float* state,
                          const float* found_inf, void* const* peer_half, int n_peers, long shard_off, ia_stream_t stream);

/* fp16 refresh of the padded MLP weight block only (the hash table is refreshed by ia_adam_step_dev) */
int ia_mlp_to_half(const float* enc_params, const float* col_params, void* mlp_h, ia_stream_t stream);
/* the same block built from the flat fp16 image of the parameters (enc_mlp_h: the first 3072 halfs of the image of
 * `encoder.params`, col_h: the 6144 halfs of `color_net.params`): with the sharded optimiser every rank holds the
 * all-gathered fp16 image while only a shard's owner holds current fp32 values. */
int ia_mlp_to_half_from_half(const void* enc_mlp_h, const void* col_h, void* mlp_h, ia_stream_t stream);
/* Sharded optimiser (reduce-scatter -> Adam on 1/G of the parameters -> all-gather of the fp16 image; the reference has
 * one replicated torch.optim.Adam, DNeRF.py:46-59,152-159): if *found_inf != 0 (this rank's LOCAL gradient overflowed,
 * ia_grad_check_finite) write a NaN into element k*shard_elems of `grads` for k < n_shards, so that after the
 * sum-reduce-scatter EVERY rank's shard fails ia_grad_check_finite and all ranks skip the step together. */
int ia_grad_poison_shards(float* grads, long shard_elems, int n_shards, const float* found_inf, ia_stream_t stream);

/* Training batches sampled on the device from device-resident frames (datasets/peoplesnapshot.py:99-151, custom.py:97-149,
 * utils/sampler.py; DESIGN.md §5.7).  Frames: images [F][H][W][3] uint8 (as decoded, cv2's channel order), masks [F][H][W]
 * fp32, ray tables rays_o / rays_d [H][W][3] (shared by the frames), near_far [F][2].
 *
 * ia_frame_index_build (once per frame set) builds, per frame, three bit sets with per-word exclusive prefix counts in a
 * caller buffer of ia_frame_index_bytes(F, H, W, patch) bytes (0 for invalid sizes):
 *   mask   {i : mask[i] != 0} over flat pixels i = y*W + x;
 *   edge   EdgeSampler's band: i such that the flat window [i - k/2, i - k/2 + k - 1] clipped to [0, H*W) holds two different
 *          values (cv2.erode / cv2.dilate of mask.reshape(-1), an (H*W) x 1 image; horizontal only, wrapping across rows).
 *          edge_kernel k = 0: empty;
 *   centre PatchSampler's valid corners (r, c), 0 <= r < H-P, 0 <= c < W-P, as r*(W-P) + c, where m'[r + P/2][c + P/2] > 0;
 *          m' is the mask, or with dilate = d > 0 its max over rows / columns y - d/2 .. y - d/2 + d - 1 inside the frame.
 *          patch P = 0: no centre set (P even, P < H, P < W otherwise).
 * counts [F][3] int64 receives the three set sizes.  edge_kernel <= 1024, dilate <= 256.
 *
 * A 32-bit random word selects element (word * count) >> 32 (64-bit product) of a set of size count.
 *   ia_sample_edge: rays t < num_mask from the mask set, then num_edge from the edge band, then num_rand uniform over the
 *     H*W pixels; words [n] (n = num_mask + num_edge + num_rand).  words NULL (index may be NULL): ray t is pixel t, the
 *     full frame (num_mask = num_edge = 0, num_rand = H*W).  `patch` is the P the index was built with.
 *   ia_sample_patch: num_patch (<= 1024) patches of P x P; words [1 + 2*num_patch].  Mask branch iff words[0] / 2^32 <
 *     ratio_mask: distinct centres by Floyd's algorithm (for j = C-n .. C-1, t from words[1 + j - (C-n)] over [0, j]; t,
 *     or j when t was taken, in that order).  Otherwise r from words[1 + p] over [0, H-P) and c from words[1 + n + p] over
 *     [0, W-P).  Patch p covers rows r .. r+P-1 and columns c .. c+P-1; its rays are p*P*P + dy*P + dx.
 * Per ray t from pixel i of `frame`: rgb[t] = img * m + (1 - m) * bg[t] with img = u8 / 255 (IEEE division, no
 * contraction), alpha[t] = m, rays_o/rays_d[t] = the tables at i, bg_color[t] = bg[t] (bg NULL: 1), near/far[t] =
 * near_far[frame].  A ray drawn from an empty set (or a mask-branch patch with fewer than num_patch centres) gets NaN in
 * every output. */
size_t ia_frame_index_bytes(int F, int H, int W, int patch);
int ia_frame_index_build(const float* masks, int F, int H, int W, int edge_kernel, int patch, int dilate, void* index,
                         size_t nbytes, int64_t* counts, ia_stream_t stream);
int ia_sample_edge(const uint8_t* images, const float* masks, const float* rays_o, const float* rays_d, const float* near_far,
                   int F, int H, int W, const void* index /*nullable with words*/, int patch, int frame, int num_mask,
                   int num_edge, int num_rand, const uint32_t* words /*nullable*/, const float* bg /*nullable*/, float* rgb,
                   float* alpha, float* out_rays_o, float* out_rays_d, float* bg_color, float* near, float* far,
                   ia_stream_t stream);
int ia_sample_patch(const uint8_t* images, const float* masks, const float* rays_o, const float* rays_d, const float* near_far,
                    int F, int H, int W, const void* index, int frame, int num_patch, int patch, double ratio_mask,
                    const uint32_t* words, const float* bg, float* rgb, float* alpha, float* out_rays_o, float* out_rays_d,
                    float* bg_color, float* near, float* far, ia_stream_t stream);

/* Test-split evaluation (DNeRF.py:225-239 and eval.py:93-118; DESIGN.md §3, §5.8).
 *
 * ia_test_panel: pred, gt [F][H][W][3] fp32 -> panel [F][H][3W][3] uint8, row y of frame f = [q(gt) | q(pred) | JET[e]] in
 * the inputs' channel order (cv2's BGR, as the frames are stored), the image the reference's test_step writes.
 *   q(v) = saturate_u8(rint(float32(v * 255))), rint rounding half to even, as cv2.imwrite converts float images; NaN, and
 *          products at or above 2^31 (+inf included), give 0 (cv2 on x86-64; aarch64 builds of cv2 saturate those to 255).
 *   e    = trunc(float32(float32(sqrt((d0^2 + d1^2) + d2^2)) / float32(sqrt 3)) * 255) with d = pred - gt, every operation
 *          in float32 without contraction (numpy 1.x promotion of DNeRF.py:230).  Where numpy's astype(uint8) is undefined
 *          the index saturates: e >= 256 -> 255, NaN -> 0.
 *   JET  = OpenCV's COLORMAP_JET (instantavatar_b200/csrc/ia_jet_lut.cuh).
 * F * H * W < 2^31.
 *
 * ia_image_metrics: per frame f of two uint8 stacks a, b [F][H][W][3] (pixel bytes contiguous; byte strides per frame and per
 * row, so the pred and gt thirds of a panel are read in place):
 *   sse[f]     = sum over the 3*H*W bytes of (a - b)^2, exact;
 *   ssim_fx[f] = sum over the 3 channels and the (H-10)*(W-10) valid 11 x 11 windows of rint(s * 2^32) (half to even), s the
 *                SSIM of torchmetrics' StructuralSimilarityIndexMeasure(data_range=1) at that window, evaluated in float64:
 *                x = (double)((float)k / 255.0f); the five maps x, y, x*x, y*y, x*y filtered horizontally, then vertically,
 *                each a sequential sum over t = 0..10 of taps[t] * v; sigma_x = E[xx] - mx*mx (no clamp), likewise sigma_y,
 *                sigma_xy; s = ((2*(mx*my) + c1) * (2*sigma_xy + c2)) / ((mx*mx + my*my + c1) * (sigma_x + sigma_y + c2)),
 *                c1 = 0.01^2, c2 = 0.03^2.
 *   taps: HOST array of 11 doubles (torchmetrics' float32 Gaussian, sigma 1.5, widened).  sse, ssim_fx: [F] int64 (device),
 *   overwritten.  IA_EINVAL: H or W < 11 (no valid window), H*W > 2^28 (the bound that keeps 3*H*W*2^32 < 2^63), F > 65535,
 *   a row stride below 3*W, or (F > 1) a frame stride below (H-1)*row_stride + 3*W. */
int ia_test_panel(const float* pred, const float* gt, int F, int H, int W, uint8_t* panel, ia_stream_t stream);
int ia_image_metrics(const uint8_t* a, long frame_stride_a, long row_stride_a, const uint8_t* b, long frame_stride_b,
                     long row_stride_b, int F, int H, int W, const double* taps, int64_t* sse, int64_t* ssim_fx,
                     ia_stream_t stream);

/* GIF palettes of animation frames (animate.py:117-118, novel_view.py:127-128; DESIGN.md §3.2, §5.9).
 *
 * ia_gif_quantize: rgba [F][H][W][4] uint8 -> per frame f its own palette [f][256][3] (R, G, B), index [f][H][W] and
 * n_colors[f] <= 256.  Channels (0, 1, 2) are read as R, G, B; swap_rb = 1 reads (2, 1, 0), for frames in cv2's BGRA order.
 * Alpha is ignored.  Integer-only median cut, so results are exact:
 *   1. histogram: per bin (r>>3, g>>3, b>>3) the pixel count and the exact channel sums;
 *   2. one box, the bounding box (in bins) of the occupied bins;
 *   3. while fewer than 256 boxes: take the box with the most pixels among boxes wider than one bin (ties: lowest index;
 *      stop if none); split its longest side in bins (ties: r, g, b) at the smallest plane c in [lo, hi-1] with
 *      2 * (pixels at or below c) >= the box's pixels (c = hi-1 if none); the lower half keeps the index, the upper half
 *      is appended; both shrink to the bounding box of their occupied bins;
 *   4. palette entry k = (2 * sum + n) / (2n) per channel over the box's n pixels (integer division); entries >= n_colors
 *      are 0;
 *   5. index = the lowest k < n_colors minimising the integer squared RGB distance to the pixel's exact colour.
 * workspace: device, 16-byte aligned, ia_gif_quantize_workspace_bytes(F) bytes (512 KB per frame).  rgba 4-byte aligned.
 * IA_EINVAL: F outside [0, 65535], H or W < 1, H*W > 2^24, a short workspace, a NULL pointer (F > 0). */
size_t ia_gif_quantize_workspace_bytes(int F);
int ia_gif_quantize(const uint8_t* rgba, int F, int H, int W, int swap_rb, uint8_t* palette, uint8_t* index, int* n_colors,
                    void* workspace, size_t workspace_bytes, ia_stream_t stream);

/* Batched SMPL forward and reverse mode for fitting F frames of poses to 2D keypoints: the keypoint stage of
 * refine-smpl.py (scripts/custom/refine-smpl.py:166-189; DESIGN.md §3, §5.10).  fp32 throughout.
 *
 * Model (device, fp32, the layouts of instantavatar_b200.deformers.smpl.SMPL): v_template [V][3], shapedirs [V][3][10],
 * posedirs [207][3V], J_regressor [24][V] (dense), lbs_weights [V][24], parents [24] int32 (-1 for the root).
 * params: one flat vector [10 + 75F] = betas [10] | global_orient [F][3] | body_pose [F][69] | transl [F][3]; betas are
 * shared by every frame.  workspace: device, 16-byte aligned, ia_smpl_fit_workspace_bytes(V, F) bytes (0 for invalid
 * sizes).  No host synchronisation; two calls on the same input give bit-identical results (fixed-order reductions).
 *
 * ia_smpl_fit_forward: verts [F][V][3], joints [F][35][3] (the 24 posed joints, then the vertices vertex_ids [11], host),
 *   A [F][24][4][4] (the bone transforms with transl, as smplx returns them); each output nullable.
 * ia_smpl_fit_objective: loss [1] (device, nullable) and grad [10 + 75F] (written, in the layout of params) of
 *     mean_{f, b selected} m_fb |kp_fb - uv_fb|  +  mean_{f < F-1, v} |verts[f+1][v] - verts[f][v]|
 *   where BODY25 joint b is smplx joint joint_map[b] (0..23 posed joint, 24 + k vertex joint k), uv is its projection by
 *   proj = K . E[:3] (host, [3][4] row-major): uv = p[:2] / p[2], p = proj[:, :3] x + proj[:, 3]; m_fb = conf_fb > threshold;
 *   the first mean is over F * (number of selected b), masked entries included.  A residual of exactly zero contributes a
 *   zero gradient.  keypoints [F][25][3] (device; u, v, confidence).  IA_EINVAL: F < 2, no selected joint, a joint_map
 *   entry outside [0, 35), a vertex id outside [0, V). */
typedef struct {
    const float* v_template;
    const float* shapedirs;
    const float* posedirs;
    const float* J_regressor;
    const float* lbs_weights;
    const int* parents;
    int n_verts;
} IaSmplModel;

typedef struct {
    const float* keypoints;   /* device [F][25][3] */
    const float* proj;        /* host [3][4] */
    const int* joint_map;     /* host [25] */
    const int* select;        /* host [25], non-zero: in the keypoint mean */
    const int* vertex_ids;    /* host [11] */
    float threshold;
} IaKeypointFit;

size_t ia_smpl_fit_workspace_bytes(int n_verts, int F);
int ia_smpl_fit_forward(const IaSmplModel* model /*[host]*/, const float* params, int F, const int* vertex_ids /*[host]*/,
                        void* workspace, size_t workspace_bytes, float* verts, float* joints, float* A, ia_stream_t stream);
int ia_smpl_fit_objective(const IaSmplModel* model /*[host]*/, const IaKeypointFit* fit /*[host]*/, const float* params, int F,
                          void* workspace, size_t workspace_bytes, float* loss, float* grad, ia_stream_t stream);

/* Hard rasterisation and headlight shading of F posed meshes that share one face list, composited over the frames:
 * visualize-SMPL.py's overlay video (DESIGN.md §3.4, §5.11).  fp32 throughout.
 *
 * verts [F][V][3] (device, world space), faces [NF][3] int32 (device; a face with an index outside [0, V) is not drawn),
 * K [3][3] and E [4][4] (HOST, row-major; the cameras.npz intrinsic / extrinsic, only E's first three rows are read).
 * workspace: device, 16-byte aligned, ia_raster_workspace_bytes(F, V, NF) bytes (0 for invalid sizes), shared by both
 * calls.  No host synchronisation; two calls on the same input give bit-identical results.
 *
 * ia_raster: per frame f and pixel (row r, column j), sampled at the image point (u, v) = (j, r) with
 *   [u v 1]^T ~ K (R x + t): face_id [F][H][W] int32 (-1: none), depth [F][H][W] (camera-space z = 1 / sum_i b_i / z_i of
 *   the screen-space barycentrics b_i; 0 where face_id = -1) and bary [F][H][W][2] (the perspective-correct barycentrics of
 *   faces[id][1] and faces[id][2]; 8-byte aligned).  Coverage: all three edge functions >= 0 at the sample point after
 *   orienting the face (both windings drawn).  Visibility: the smallest depth, ties to the lowest face index.  Not drawn: a
 *   face with a vertex at camera z <= 0.01, a face of zero screen area, a fragment with z > 8.
 * ia_shade_composite: frames [F][H][W][3] uint8 (device, BGR, in place): each pixel with a face becomes
 *   uint8(min(255, floor(255 c + 0.5))), c = albedo (ka + kd |n . l|), with n the perspective-correct interpolation of the
 *   normalised vertex normals (area-weighted face normals summed in the order of the vertex -> face CSR csr_offsets [V+1],
 *   csr_faces [csr_offsets[V]], device int32) and l the unit view ray of the pixel; face_id and bary as ia_raster wrote them.
 * IA_EINVAL: F outside [0, 65535], a negative V or NF, H or W outside [1, 16384], a singular K, a short workspace, a NULL
 * pointer. */
size_t ia_raster_workspace_bytes(int F, int n_verts, int n_faces);
int ia_raster(const float* verts, int F, int n_verts, const int* faces, int n_faces, const float* K /*[host]*/,
              const float* E /*[host]*/, int H, int W, void* workspace, size_t workspace_bytes, int* face_id, float* depth,
              float* bary, ia_stream_t stream);
int ia_shade_composite(const float* verts, int F, int n_verts, const int* faces, int n_faces, const int* csr_offsets,
                       const int* csr_faces, const float* K /*[host]*/, const float* E /*[host]*/, int H, int W,
                       const int* face_id, const float* bary, void* workspace, size_t workspace_bytes, uint8_t* frames,
                       ia_stream_t stream);
/* ia_vertex_normals: normals [V][3] of one mesh verts [V][3], computed by ia_shade_composite's normal pass (area-weighted
 * face normals summed in csr order, normalised; 0 where they cancel), so bit-identical to the normals it shades with.
 * V = 0: nothing is done; a negative V or NF, a NULL pointer: IA_EINVAL. */
int ia_vertex_normals(const float* verts, int n_verts, const int* faces, int n_faces, const int* csr_offsets,
                      const int* csr_faces, float* normals, ia_stream_t stream);

/* Mask clean-up of a custom sequence: the per-frame body of scripts/custom/extract-largest-connected-components.py
 * (cv2.threshold(img, 0, 255, THRESH_BINARY), morphologyEx MORPH_OPEN then MORPH_CLOSE with a 5x5 all-ones kernel,
 * connectedComponentsWithStats(connectivity=8), the arg-max area and img[~mask] = 0) for F frames of one size H x W
 * (DESIGN.md §3.5, §5.12).
 *
 * masks [F][H][W] uint8: the grayscale values; v > 0 is foreground.  Erosion reads pixels outside the image as
 * foreground, dilation as background (cv2's default border).  mask_out [F][H][W] uint8 receives 255 on the kept
 * component and 0 elsewhere.  images / images_out [F][H][W][3] uint8 are both NULL or both set; images_out may alias
 * images and receives the image with every pixel outside the kept component zeroed.  stats [F][2] int32 receives the
 * number of 8-connected components after the closing (cv2's num_labels - 1) and the kept component's area.  The largest
 * area is kept; an exact tie goes to the component whose first pixel in raster order (lowest y*W + x) is lowest.  A
 * frame with no foreground after the closing gets an all-zero mask and image and a kept area of 0.
 * workspace: device, 256-byte aligned, ia_mask_workspace_bytes(F, H, W) bytes (0 for F = 0 and invalid sizes), about
 * 12 bytes a pixel.  No host synchronisation; two calls on the same input give identical results.
 * IA_EINVAL: H or W < 1, F < 0, F*H*W >= 2^31, a short workspace, a NULL pointer, one of images / images_out NULL.  F = 0
 * does nothing. */
size_t ia_mask_workspace_bytes(int F, int H, int W);
int ia_mask_largest_component(const uint8_t* masks, int F, int H, int W, uint8_t* mask_out, const uint8_t* images,
                              uint8_t* images_out, int* stats, void* workspace, size_t workspace_bytes, ia_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* IA_B200_H */
