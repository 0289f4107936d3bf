/*
 * goslam_b200.h — C-ABI of libgoslam_b200.so (sm_90a).
 *
 * One entry point per operator of GO-SLAM's per-keyframe dense-update path.  Every
 * function takes raw DEVICE pointers + shapes + a cudaStream_t (passed as void*) and
 * returns 0 on success or a negative GOSLAM_E* code; nothing is retained, nothing is
 * allocated (callers hand in workspaces sized by the *_workspace_bytes helpers), no
 * host<->device synchronisation happens inside.  No torch types cross this boundary.
 *
 * Each entry cites the reference interface (file:line under /root/reference) it
 * replaces.  The Python shim `droid_backends` (go-slam_b200/droid_backends.py) binds
 * these through ctypes under the reference's own function names.
 */
#ifndef GOSLAM_B200_H_
#define GOSLAM_B200_H_

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GOSLAM_OK            0
#define GOSLAM_EINVAL       (-1)  /* bad shape / argument                         */
#define GOSLAM_ELAUNCH      (-2)  /* cudaGetLastError() != cudaSuccess after launch */
#define GOSLAM_EWORKSPACE   (-3)  /* workspace too small                          */
#define GOSLAM_EUNSUPPORTED (-4)  /* e.g. training-only backward entry points     */

/* element types of correlation volumes / feature maps */
#define GOSLAM_F32 0
#define GOSLAM_F16 1

/* library identification; returns e.g. 100 for "1.0.0" and the SM arch compiled for */
int goslam_version(void);
int goslam_sm_arch(void);
const char* goslam_strerror(int code);
/* cudaGetErrorString of the CUDA error behind this thread's most recent GOSLAM_ELAUNCH ("" if none) */
const char* goslam_last_cuda_error(void);

/* ------------------------------------------------------------------------------------
 * Correlation volume — radius-r bilinear window lookup, one pyramid level.
 * Replaces droid_backends.corr_index_forward  (src/lib/droid.cpp:170-178,
 * src/lib/correlation_kernels.cu:19-70,126-155).
 *   volume [N,h1,w1,h2,w2] (f16|f32), coords [N,2,h1,w1] f32 (x then y),
 *   corr   [N,2r+1,2r+1,h1,w1] same dtype as volume, x-offset-major, fully overwritten.
 * A tap outside the level adds nothing (the reference's within_bounds).  So a NaN or infinite coordinate,
 * whose bilinear weights are NaN, gives NaN in the outputs with a tap inside the level and 0 in the others
 * (floor(NaN) converts to 0, an infinite or huge floor saturates and leaves every tap outside).  This holds for
 * every lookup entry point below.
 * ---------------------------------------------------------------------------------- */
int goslam_corr_index_forward(const void* volume, int dtype, const float* coords,
                              void* corr, int N, int h1, int w1, int h2, int w2,
                              int radius, void* stream);

/* Fused 4-level form of CorrBlock.__call__ (src/modules/corr.py:43-53): level i samples
 * pyramid[i] (dims h2>>i, w2>>i, floor) at coords/2^i and writes channels
 * [i*(2r+1)^2, (i+1)*(2r+1)^2) of out [N, L*(2r+1)^2, h1, w1].
 *   coords_hw2 [N,h1,w1,2] f32 — the *un-permuted* reproject output (x,y interleaved).
 *   pyramid[L] device pointers to the L level volumes (host array of L pointers). */
int goslam_corr_pyramid_lookup(const void* const* pyramid, int dtype, int num_levels,
                               const float* coords_hw2, void* out,
                               int N, int h1, int w1, int h2, int w2, int radius,
                               void* stream);

/* ------------------------------------------------------------------------------------
 * Correlation volume — all-pairs build + 2x2 average-pool pyramid.
 * Replaces CorrBlock.__init__/CorrBlock.corr (src/modules/corr.py:25-41,67-76):
 *   corr[n] = (fmap1[n]/4)^T (fmap2[n]/4)  -> level0 [N,h,w,h,w]; level i+1 = avg_pool2d(level i,2,2).
 * CUDA-core build in the reference's row-major layout:
 *   fmap1,fmap2 [N,D,h,w] (channel-major, as DepthVideo.fmaps stores them), dtype GOSLAM_F16 | GOSLAM_F32;
 *   levels[L] output pointers of the same dtype, level i dims [N,h,w,h>>i,w>>i].
 * The tensor-core build is goslam_corr_pool_build below. */
int goslam_corr_build(const void* fmap1, const void* fmap2, int dtype, void* const* levels,
                      int num_levels, int N, int D, int h, int w, void* stream);
/* Video-level form of FactorGraph.add_factors' correlation build (src/factor_graph.py:106-114):
 * the per-frame feature maps are kept K-major AND PRE-SCALED BY 1/4 in half — the reference's
 * `fmap / 4.0` (src/modules/corr.py:71-72) — as [F = buffer*rig, h*w, D] f16, converted ONCE when a
 * keyframe is inserted by goslam_fmaps_to_kmajor from DepthVideo.fmaps' [F, D, h, w], and the
 * kernel indexes them per edge on the device: slot1 = rig*ii[e], slot2 = rig*jj[e] + (ii[e]==jj[e])
 * — no gathered [N,D,h,w] copies, no per-edge re-layout.  Tensor-core kernel only (D == 128, w <= 128). */
int goslam_fmaps_to_kmajor(const void* fmaps, void* out, int F, int D, int h, int w, void* stream);

/* Slot-pool build and lookup: the edge dimension of the volume is a POOL of `capacity` slots that the
 * factor graph allocates once; edge e of a block lives in slot slots[e] (int32, device).  Makes
 * CorrBlock.cat / CorrBlock.__getitem__ (src/modules/corr.py:55-65, hit on every add_factors /
 * rm_factors, src/factor_graph.py:114,149) an edit of the slot table instead of a copy of the
 * whole pyramid.  slots == NULL means identity (slot e = edge e).
 *   levels[L]: pool buffers, f16.
 *
 * layout: GOSLAM_LAYOUT_ROWMAJOR = the reference's [slot,h,w,h>>i,w>>i];
 *         GOSLAM_LAYOUT_TILED    = levels 0 and 1 stored as 4x4-element (32-byte = one DRAM sector)
 *         tiles, tile-row-major inside each source pixel's plane, planes padded to whole tiles; levels 2
 *         and 3 as one padded piece per 8-row band of level 0.  Padding contents are unspecified (the
 *         build pools the coarser levels' padding from the finer level's, and skips some of it); the
 *         lookup never reads them into a result.  Nothing in the
 *         reference outside CorrBlock reads the pyramid, so its layout is private to build + lookup:
 *         the tiled form turns the build's per-thread output into one 128-byte run and cuts the sectors
 *         an 8x8 lookup window touches from ~11.5 to ~7.6.  goslam_corr_level_plane_elems gives the
 *         per-source-pixel plane size (f16 elements) of a level: buffer i holds capacity * h*w *
 *         plane_elems(i) elements.
 * goslam_corr_pool_build always writes the tiled layout; goslam_corr_pool_lookup reads either (the
 * row-major form serves caller-owned volumes and goslam_corr_build's output, f16 or f32). */
#define GOSLAM_LAYOUT_ROWMAJOR 0
#define GOSLAM_LAYOUT_TILED 1
size_t goslam_corr_level_plane_elems(int level, int layout, int h, int w);
int goslam_corr_pool_build(const void* fmaps_kmajor, int F, int rig, const int64_t* ii,
                           const int64_t* jj, const int* slots, void* const* levels,
                           int num_levels, int N, int D, int h, int w, void* stream);
int goslam_corr_pool_lookup(const void* const* pyramid, int dtype, int num_levels, const int* slots,
                            int capacity, int layout, const float* coords_hw2, void* out, int N,
                            int h1, int w1, int h2, int w2, int radius, void* stream);

/* ------------------------------------------------------------------------------------
 * On-the-fly windowed correlation (no volume).
 * Replaces droid_backends.altcorr_forward (src/lib/droid.cpp:193-203,
 * src/lib/altcorr_kernel.cu:27-149,290-319).
 *   fmap1 [B,H,W,C] f32, fmap2 [B,H2,W2,C] f32 (NHWC), coords [B,S,H,W,2] f32,
 *   corr [B,S,(2r+1)^2,H,W] f32, channel = xoff*(2r+1)+yoff, fully overwritten. */
int goslam_altcorr_forward(const float* fmap1, const float* fmap2, const float* coords,
                           float* corr, int B, int S, int H, int W, int H2, int W2,
                           int C, int radius, void* stream);

/* AltCorrBlock.__call__ in one launch (src/modules/corr.py:97-145, one coordinate set per edge):
 *   pyramid[l] = [F, H>>l, W>>l, C] f16 NHWC, the reference's AltCorrBlock.pyramid (fmaps/4,
 *   avg-pooled), shared by all edges; ii, jj [N] int64 index F (the reference passes rig*ii and
 *   rig*jj + (ii==jj)); coords [N,H,W,2] f32 at level-0 resolution (scaled by 2^-l inside);
 *   out [N, L*(2r+1)^2, H, W] f32, level-major, x-offset-major inside a level. */
int goslam_altcorr_pyramid(const void* const* pyramid, int num_levels, const float* coords,
                           const int64_t* ii, const int64_t* jj, float* out, int N, int H, int W,
                           int C, int radius, void* stream);

/* ------------------------------------------------------------------------------------
 * Geometry kernels of droid_backends (src/lib/droid.cpp:120-160,220-225).
 *   poses [num,7] f32 (tx,ty,tz,qx,qy,qz,qw); disps [num,ht,wd] f32; intrinsics [4]
 *   f32 (fx,fy,cx,cy); ii,jj int64.
 *   projmap, reproject, reproject_motion and depth_filter launch one grid row per edge and
 *   iproj one per frame: K (num for iproj) above 65535 returns GOSLAM_EINVAL before any CUDA
 *   call.
 * ---------------------------------------------------------------------------------- */
/* frame_distance (src/lib/droid_kernels.cu:518-657,1438-1460): dist [K] f32.
 * Reduction order reproduces the reference's 256-thread strided sum + 128/64/32..1 tree
 * so thresholded edge lists are bit-identical. */
int goslam_frame_distance(const float* poses, const float* disps, const float* intrinsics,
                          const int64_t* ii, const int64_t* jj, float* dist,
                          int K, int ht, int wd, float beta, void* stream);
/* DepthVideo.distance(bidirectional=True) (src/depth_video.py:233-245): 0.5 * (d(i->j) + d(j->i)) in one
 * launch instead of two launches and two elementwise kernels; bit-identical to that form. */
int goslam_frame_distance_bidir(const float* poses, const float* disps, const float* intrinsics,
                                const int64_t* ii, const int64_t* jj, float* dist, int K, int ht,
                                int wd, float beta, void* stream);
/* Banded bidirectional distance grid for Backend.ba (src/backend.py:31-44) without index tensors:
 * dist [r1-r0, c1-c0] f32 row-major, entry (i, j) (frames i in [r0, r1), j in [c0, c1)) is
 * goslam_frame_distance_bidir of the pair, bit for bit, where j - i <= k and +inf elsewhere.
 * Backend.ba reads nothing else with k = -radius (dense) or k = 2 - radius (loop closure).
 * The poses of frames [0, max(r1, c1)) are first copied into the workspace on `stream`, so
 * every pair sees the poses as they were when the call reached the stream.
 *   Empty ranges are a no-op; negative starts or ends below starts return GOSLAM_EINVAL, as do
 *   null tensors for a non-empty grid.
 *   workspace: goslam_frame_distance_grid_workspace_bytes(r0, r1, c0, c1) (0 for empty ranges). */
size_t goslam_frame_distance_grid_workspace_bytes(int r0, int r1, int c0, int c1);
int goslam_frame_distance_grid(const float* poses, const float* disps, const float* intrinsics,
                               int r0, int r1, int c0, int c1, int k, int ht, int wd, float beta,
                               float* dist, void* workspace, size_t workspace_bytes, void* stream);
/* projmap (src/lib/droid_kernels.cu:427-516,1463-1488): coords [K,ht,wd,3] (3rd
 * component left zero, as the reference does), valid [K,ht,wd,1]. */
int goslam_projmap(const float* poses, const float* disps, const float* intrinsics,
                   const int64_t* ii, const int64_t* jj, float* coords, float* valid,
                   int K, int ht, int wd, void* stream);
/* iproj (src/lib/droid_kernels.cu:779-850,1518-1541): points [num,ht,wd,3]. */
int goslam_iproj(const float* poses, const float* disps, const float* intrinsics,
                 float* points, int num, int ht, int wd, void* stream);
/* depth_filter (src/lib/droid_kernels.cu:661-775,1491-1515): counter [K,ht,wd],
 * fully overwritten (zeroed inside). */
int goslam_depth_filter(const float* poses, const float* disps, const float* intrinsics,
                        const int64_t* ix, const float* thresh, float* counter,
                        int K, int num, int ht, int wd, void* stream);
/* Multiview filter: one pass of MultiviewFilter.forward (src/multiview_filter.py:98-170) over
 * the first T keyframes at full resolution ht x wd, in two calls on one stream.
 *   compute: poses [T,7] (w2c snapshot, for depth_filter's votes), poses_world [T,7]
 *     (w2w * SE3(poses).inv(), for iproj's points), disps [T,ht,wd], intrinsic [4] (scaled to
 *     full resolution), filter_thresh, visible_num, kernel_size (0 = 'inf', < 2 = no dilation,
 *     else a box of (k/2)*2+1, radius at most 15).  Writes only the workspace.
 *   commit: reads the same poses / disps and the workspace; only if the mask1 count is >= 100
 *     and the final point set is non-empty, it adds pose_dist(poses_filtered, poses) to
 *     update_priority[:T], then writes poses_filtered[:T], disps_filtered[:T], mask_filtered[:T]
 *     (0/1 floats), filtered_id[0] = T and bound [3,2].  Always writes
 *     status[4] = {mask1 count, extended count, final count, committed}.
 * workspace_bytes returns 0 for invalid sizes. */
size_t goslam_mvfilter_workspace_bytes(int T, int ht, int wd);
int goslam_mvfilter_compute(const float* poses, const float* poses_world, const float* disps,
                            const float* intrinsic, float filter_thresh, int visible_num,
                            int kernel_size, int T, int ht, int wd, void* workspace,
                            size_t workspace_bytes, void* stream);
int goslam_mvfilter_commit(const float* poses, const float* disps, const void* workspace,
                           size_t workspace_bytes, int T, int ht, int wd, float* poses_filtered,
                           float* disps_filtered, float* mask_filtered, float* update_priority,
                           int* filtered_id, float* bound, int64_t* status, void* stream);
/* reproject = pops.projective_transform(jacobian=False) as called by DepthVideo.reproject
 * (src/depth_video.py:207-217, src/geom/projective_ops.py:114-144) with the lietorch SE3
 * algebra restated from src/lib/droid_kernels.cu:58-107.  intrinsics_all [num,4] (per
 * frame, as DepthVideo.intrinsics); coords [K,ht,wd,2], valid [K,ht,wd,1]. */
int goslam_reproject(const float* poses, const float* disps, const float* intrinsics_all,
                     const int64_t* ii, const int64_t* jj, float* coords, float* valid,
                     int K, int ht, int wd, void* stream);
/* reproject + the motion features FactorGraph.update feeds the update operator
 * (src/factor_graph.py:202-206): motion [K,4,ht,wd] = clamp(cat([coords1 - coords0, target - coords1]),
 * -64, 64) with coords0 the pixel grid and target [K,ht,wd,2] the edge's current flow target; one
 * launch instead of reproject + 5 elementwise kernels.  valid may be NULL. */
int goslam_reproject_motion(const float* poses, const float* disps, const float* intrinsics_all,
                            const int64_t* ii, const int64_t* jj, const float* target, float* coords,
                            float* valid, float* motion, int K, int ht, int wd, void* stream);

/* ------------------------------------------------------------------------------------
 * Dense bundle adjustment.  Replaces droid_backends.ba (src/lib/droid.cpp:88-117,
 * src/lib/droid_kernels.cu:1314-1434 + kernels :176-424,:854-1115 + the host Eigen
 * Schur/LLT :1117-1311).  poses and disps are updated IN PLACE.
 *   targets,weights [N,2,ht,wd] f32; disps_sens [num,ht,wd].
 *   eta [eta_rows,ht,wd] f32: eta_rows == M = |unique([t0,t1) U ii)| (rows in sorted frame order —
 *   the reference's `damping[unique(cat(arange(t0,t1), ii))]`, src/factor_graph.py:236-238),
 *   eta_rows == 1 (one row, broadcast) or eta_rows == -num (negative: eta is [num,ht,wd] indexed
 *   by FRAME id — the form the sharded driver uses, where every rank has its own slot order).
 *   Any other row count is a caller bug (the reference raises a broadcast error,
 *   src/lib/droid_kernels.cu:1397): the call leaves poses/disps untouched, dx = 0, status 2.
 *   dx_out [t1-t0,6] (nullable), dz_out [num,ht*wd] indexed by FRAME id (nullable).
 *   status_out: device int[iterations] (nullable), 0 = solved, 1 = factorisation failed
 *   (then dx = 0 for that iteration, like src/lib/droid_kernels.cu:1207-1210), 2 = eta row count
 *   mismatch (see above).
 * Limits: num <= 4096 frames.
 * ---------------------------------------------------------------------------------- */
size_t goslam_ba_workspace_bytes(int N, int num, int ht, int wd, int t0, int t1);
int goslam_ba(float* poses, float* disps, const float* intrinsics, const float* disps_sens,
              const float* targets, const float* weights, const float* eta, int eta_rows,
              const int64_t* ii, const int64_t* jj, int N, int num, int ht, int wd,
              int t0, int t1, int iterations, float lm, float ep, int motion_only,
              float* dx_out, float* dz_out, int* status_out,
              void* workspace, size_t workspace_bytes, void* stream);

/* Multi-GPU split form of one BA iteration (edges sharded by source frame ii; SURVEY §8e):
 *   phase 1  linearise local edges and accumulate the local reduced system
 *            Hred [6P*6P] f64 + bred [6P] f64 into `system` (caller all-reduces it),
 *   phase 2  damp + factorise + back-substitute + retract with the reduced system.
 * goslam_ba == phase1 + phase2 per iteration on one GPU. */
size_t goslam_ba_system_doubles(int t0, int t1);
int goslam_ba_phase1(const float* poses, const float* disps, const float* intrinsics,
                     const float* disps_sens, const float* targets, const float* weights,
                     const float* eta, int eta_rows, const int64_t* ii, const int64_t* jj,
                     int N, int num, int ht, int wd, int t0, int t1, int motion_only,
                     double* system, void* workspace, size_t workspace_bytes, void* stream);
int goslam_ba_phase2(float* poses, float* disps, const double* system,
                     int N, int num, int ht, int wd, int t0, int t1,
                     float lm, float ep, int motion_only, int owner_lo, int owner_hi,
                     float* dx_out, float* dz_out, int* status_out,
                     void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------
 * The split form over PEER MEMORY (one node, NVLink / NVSwitch): what SURVEY 8e asks NCCL for — one all-reduce of the
 * reduced camera system and one all-gather of the owned inverse-depth rows per Gauss-Newton iteration — done by the
 * BA kernels themselves.  Every rank keeps its partial system, its replica of disps and a row of flag words in buffers
 * the other ranks have mapped (goslam_ipc_open on a CUDA IPC handle; the host side exchanges the handles once).
 *   phase1_peers: waits (on the device) until every rank has finished iteration epoch-1, linearises the local edges,
 *                 leaves the partial system in system[rank] and raises flag [rank] on every rank.
 *   phase2_peers: the solve kernel waits for all flags and sums the partial systems IN RANK ORDER while it loads the
 *                 matrix into shared memory (every rank factors bit-identical numbers), retracts the poses, and the
 *                 back-substitution writes the rows of frames [owner_lo, owner_hi) into every replica of disps; then
 *                 raises flag [world + rank] on every rank.
 * No host synchronisation, no collective library call.  A wait that sees no progress for ~2 s sets *timeout = 1 and
 * continues (a dead peer must not hang the GPU); the caller checks it.
 *   flags[r]: u32 [2 * world] in rank r's memory, zero before the first call; epoch: >= 1, +1 per iteration, the same
 *   on all ranks, never reused.  disps[rank] is the local replica the kernels read and update. */
typedef struct goslam_ba_peers {
  int world, rank;
  double* system[8];
  float* disps[8];
  unsigned* flags[8];
  unsigned epoch;
  int* timeout;            /* local device int (may be NULL) */
} goslam_ba_peers;
int goslam_ba_phase1_peers(const float* poses, const float* intrinsics, const float* disps_sens,
                           const float* targets, const float* weights, const float* eta, int eta_rows,
                           const int64_t* ii, const int64_t* jj, int N, int num, int ht, int wd, int t0, int t1,
                           int motion_only, const goslam_ba_peers* peers, void* workspace, size_t workspace_bytes,
                           void* stream);
int goslam_ba_phase2_peers(float* poses, int N, int num, int ht, int wd, int t0, int t1, float lm, float ep,
                           int motion_only, int owner_lo, int owner_hi, const goslam_ba_peers* peers, float* dx_out,
                           float* dz_out, int* status_out, void* workspace, size_t workspace_bytes, void* stream);
/* stream-ordered wait until every rank has finished iteration peers->epoch (its rows are in my replica, it no longer
 * reads my partial system): what a caller puts before it touches its replica of disps outside the BA calls */
int goslam_ba_peers_wait(const goslam_ba_peers* peers, void* stream);
/* a zero-filled device allocation other processes can map (cudaMalloc + cudaIpcGetMemHandle): handle_out gets the 64-byte
 * CUDA IPC handle to send to the peers */
int goslam_peer_alloc(size_t bytes, void** ptr, void* handle_out);
int goslam_peer_free(void* ptr);
/* map / unmap a peer process's device allocation from its 64-byte CUDA IPC handle (cudaIpcOpenMemHandle) */
int goslam_ipc_open(const void* handle, void** ptr);
int goslam_ipc_close(void* ptr);

/* ------------------------------------------------------------------------------------
 * Hash-grid neural-surface ray marcher.  Replaces InstantNeuS.forward
 * (src/InstantNeuS.py:295-370) incl. tiny-cuda-nn HashGrid + FullyFusedMLP
 * (src/InstantNeuS.py:44-66,184-205), SDFNetwork.sdf + autograd normal (:97-160),
 * get_alpha (:276-293) and the compositing (:343-370).
 * ---------------------------------------------------------------------------------- */
typedef struct goslam_neus_params {
  const void*  grid;        /* f16 [total_params] tcnn HashGrid layout, 16 levels x 2 feats */
  const float* sdf_w;       /* [32,35] nn.Linear weight (row-major out x in)               */
  const float* sdf_b;       /* [32]                                                        */
  const float* color_B;     /* [3,33]  ColorNetwork._B                                     */
  const void*  mlp_w;       /* f16 tcnn FullyFusedMLP params: [64,80] | [64,64] | [16,64]  */
  float bound[6];           /* self.bound  (xmin,xmax,ymin,ymax,zmin,zmax) — normalisation */
  float rt_bound[6];        /* self.realtime_bound — in_bound mask                         */
  float inv_s;              /* exp(variance*scale_factor) clipped to [1e-6,1e6]            */
  float cos_anneal_ratio;   /* self.cos_anneal_ratio (1.0)                                 */
} goslam_neus_params;

typedef struct goslam_neus_out {
  float* color;          /* [R,3]  */
  float* depth;          /* [R,1]  */
  float* depth_variance; /* [R,1]  */
  float* normal;         /* [R,3]  */
  float* weight_sum;     /* [R,1]  */
  float* sdf;            /* [R,S]  */
  float* z_mid;          /* [R,S]  (z_vals + dists/2)                    */
  float* gradient_error; /* [1]    */
  /* optional per-sample intermediates (NULL in production; the parity tests read them to check the
   * composited outputs sample by sample): */
  float* alpha;          /* [R,S]   NeuS alpha of every sample (0 outside the bound)  */
  float* grad;           /* [R,S,3] SDF normal of every sample (0 outside the bound)  */
  float* pos;            /* [R,S,3] normalised sample position in [-1,1] (0 outside the bound) */
  /* optional, kept by the training pass for goslam_neus_*_backward: */
  float* rgb;            /* [R,S,3]  colour of every sample after the sigmoid (0 outside the bound) */
  void* mlp_in;          /* [R,S,80] f16: the colour network's input row [sin(pB) 33 | normal 3 | feat 31 | 1.0 x 13] */
  void* enc;             /* [R,S,32] f16: hash-grid encoding (0 outside the bound) */
  /* optional: int [1], set to 1 when no sample of the call lies inside realtime_bound, else 0.  Then, like the
   * reference (src/InstantNeuS.py:311-312), the first 100 samples of the call ([R,S] order) go through the network as
   * if in bound.  Pass it to the backward entries so they use the same sample set.  NULL: kept in the workspace. */
  int* fallback;
} goslam_neus_out;

size_t goslam_neus_workspace_bytes(int R, int S);
int goslam_neus_forward(const goslam_neus_params* params, const float* rays_o,
                        const float* rays_d, const float* z_vals, const float* dists,
                        int R, int S, const goslam_neus_out* out,
                        void* workspace, size_t workspace_bytes, void* stream);
/* ------------------------------------------------------------------------------------
 * Renderer backward (SURVEY 8f-3).  The reference differentiates InstantNeuS.forward with autograd + tiny-cuda-nn
 * inside Mapper.optimize_map (src/mapping.py:60-148: total_loss.backward()).  Here the training pass is
 * goslam_neus_forward with the optional per-sample outputs kept (alpha, grad, rgb, mlp_in, enc), and the backward is
 * these two kernels around the colour network's plain GEMMs (which the host mirror runs on cuBLAS):
 *
 * goslam_neus_composite_backward — per ray: compositing (weights = alpha * cumprod(1 - alpha + 1e-7)), NeuS alpha
 *   (get_alpha, src/InstantNeuS.py:276-293, incl. the clip), the colour sigmoid and the eikonal term.
 *   in : saved alpha, sdf, z_mid [R,S], rgb, grad [R,S,3]; upstream d_color [R,3], d_depth [R], d_sdf [R,S] (each may
 *        be NULL = zero) and d_gradient_error (device scalar dL/d gradient_error[0], or NULL); total_samples = the number
 *        of samples gradient_error was averaged over (R*S of the WHOLE forward call when this call covers a slice of it).
 *   out: d_mlp_out [R,S,3] (w.r.t. the colour network's first three outputs, before the sigmoid), d_sdf_out [R,S],
 *        d_grad [R,S,3] (w.r.t. the SDF normal: alpha path + eikonal), d_inv_s [1] (ACCUMULATED: zero it first).
 *   Samples the forward kept out of the network get zeros (the forward gives them constants): those outside the
 *   real-time bound, unless *fallback (the forward's goslam_neus_out.fallback; NULL = 0) forced them in.  sample0 = the
 *   index of this call's first sample within the forward call (r0 * S when this call covers rays r0..); the forced
 *   samples are the forward call's first 100.  S <= 128.
 *
 * Both backward entries decide "in bound" exactly as the forward did, from the recomputed position, fallback and
 * sample0.
 *
 * goslam_neus_grid_backward — per sample: scatters dL/d(encoding) [R*S,32] (divided by *d_enc_scale when given) and the part of dL/d(normal) [R*S,3] that
 *   flows through the hash grid into grid_grad [n_params] f32 (ACCUMULATED), and accumulates into d_w0 [35] the gradient
 *   of row 0 of sdf_layer.weight THROUGH THE NORMAL (normal = (W0[:3] + 0.5 * d enc/d u . W0[3:]) * 2/(b1-b0)), i.e. the
 *   second-order path autograd takes with create_graph=True (src/InstantNeuS.py:139-146).  The direct path
 *   (d_out^T h) is a plain GEMM left to the caller.  Positions are recomputed from the rays exactly as the forward does. */
int goslam_neus_composite_backward(const goslam_neus_params* params, const float* rays_o, const float* rays_d,
                                   const float* dists, const float* alpha, const float* rgb, const float* sdf,
                                   const float* grad, const float* z_mid, const float* d_color,
                                   const float* d_depth, const float* d_sdf, const float* d_gradient_error,
                                   const int* fallback, long long total_samples, long long sample0, int R, int S,
                                   float* d_mlp_out, float* d_sdf_out, float* d_grad, float* d_inv_s, void* stream);
int goslam_neus_grid_backward(const goslam_neus_params* params, const float* rays_o, const float* rays_d,
                              const float* z_vals, const float* dists, const int* fallback, long long sample0, int R, int S,
                              const float* d_enc, const float* d_enc_scale, const float* d_grad, float* grid_grad,
                              float* d_w0, void* stream);
/* goslam_neus_composite_backward_ex — goslam_neus_composite_backward with one more optional output: d_true_cos [R,S]
 *   (NULL = not written) = dL/d true_cos, true_cos = rays_d . normal, through get_alpha alone (0 for samples kept out of
 *   the network and where the clip stops the gradient).  Every other output is the same, bit for bit.  The ray backward
 *   takes it for the direction's direct path.
 *
 * goslam_neus_ray_backward — per ray: dL/d rays_o [R,3] and dL/d rays_d [R,3] (WRITTEN, not accumulated) of the rays of
 *   the call, for camera refinement (src/mapping.py:173-194 with mapping.BA).  For a sample at p = o + z d (z = z_vals +
 *   dists/2 carries no gradient) that went through the network, dL/dp sums four paths: sdf_layer's include_xyz columns
 *   (d_xyz [R*S,3] = d_out W_sdf[:,:3] w.r.t. the normalised position, zero on clamped axes), the hash-grid encoding to first
 *   order (d_enc [R*S,32]), the analytic normal to second order (d_grad [R*S,3] = dL/d normal, mixed partials of the
 *   trilinear interpolant on the f16 table) and the colour embedding sin(p B) (dE [R*S,40] f16, 33 columns used, as
 *   goslam_neus_mlp_backward writes it).  d_enc, d_xyz and dE are in units of *scale (NULL = 1); d_grad and d_true_cos
 *   [R*S] (from goslam_neus_composite_backward_ex) are unscaled.  Then dL/d o = sum_s dL/dp_s and dL/d d =
 *   sum_s z_s dL/dp_s + sum_s d_true_cos_s normal_s.  The per-ray sums run in a fixed order without atomics: the result is
 *   deterministic and does not depend on how the caller splits the rays.  In bound / fallback / sample0 as for the other
 *   backward entries.  S <= 128. */
int goslam_neus_composite_backward_ex(const goslam_neus_params* params, const float* rays_o, const float* rays_d,
                                      const float* dists, const float* alpha, const float* rgb, const float* sdf,
                                      const float* grad, const float* z_mid, const float* d_color, const float* d_depth,
                                      const float* d_sdf, const float* d_gradient_error, const int* fallback,
                                      long long total_samples, long long sample0, int R, int S, float* d_mlp_out,
                                      float* d_sdf_out, float* d_grad, float* d_inv_s, float* d_true_cos, void* stream);
int goslam_neus_ray_backward(const goslam_neus_params* params, const float* rays_o, const float* rays_d,
                             const float* z_vals, const float* dists, const int* fallback, long long sample0, int R, int S,
                             const float* d_enc, const float* d_xyz, const void* dE, const float* scale, const float* d_grad,
                             const float* d_true_cos, float* d_rays_o, float* d_rays_d, void* stream);
/* goslam_neus_mlp_backward — the row-wise half of the colour network's backward (tcnn FullyFusedMLP 80->64->64->16, no
 * biases, ReLU, fp16) in one pass per 32-sample warp tile on mma.sync: recomputes H1, H2 from the kept input rows,
 * dH2 = (dY W3).[H2>0], dH1 = (dH2 W2).[H1>0], dX = dH1 W1, and from dX per sample: dE = dX[:33] cos(p B) (embedding),
 * d_grad_total = d_grad + dX[33:36] (normal), d_out = [d_sdf | dX[36:67]] (sdf_layer output), h = [x | enc | 1] (sdf_layer
 * input, the 1 carries the bias gradient) and the fp16 hi/lo split of the sample positions.  Gradient operands are
 * multiplied by *scale (a power of two chosen by the caller so that fp16 does not underflow) before the cast to half;
 * every fp16 output is in scaled units, d_grad_total is unscaled f32.  Left to the caller: the weight-gradient GEMMs over
 * the sample dimension (dY8^T H2, dH2^T H1, dH1^T X, pts_hl^T dE, d_out^T h) and d_enc = d_out W_sdf[:,3:]. */
typedef struct goslam_neus_mlp_bwd_out {
  void* H1; void* H2; void* dH1; void* dH2;   /* f16 [R*S,64] */
  void* dY8;                                  /* f16 [R*S,8]  scaled dL/d(MLP output), 3 columns used */
  void* dE;                                   /* f16 [R*S,40] 33 columns used */
  void* d_out;                                /* f16 [R*S,32] */
  void* h;                                    /* f16 [R*S,40] 36 columns used */
  void* pts_hl;                               /* f16 [R*S,8]  hi(3) | lo(3) */
  float* d_grad_total;                        /* f32 [R*S,3] */
} goslam_neus_mlp_bwd_out;
int goslam_neus_mlp_backward(const goslam_neus_params* params, const void* mlp_in, const void* enc, const float* pos,
                             const float* d_mlp_out, const float* d_sdf, const float* d_grad, const float* rays_o,
                             const float* rays_d, const float* z_mid, const float* scale, int R, int S,
                             const goslam_neus_mlp_bwd_out* out, void* stream);
/* ------------------------------------------------------------------------------------
 * Mesh extraction: InstantNeuS.extract_fields / extract_geometry / extract_color (src/InstantNeuS.py:402-492).
 * The pipeline is sdf_grid -> mc_count -> (caller reads the two counts, allocates) -> mc_emit -> mesh_cull_count
 * -> (reads, allocates) -> mesh_cull_emit -> neus_vertex_color.  Pointers are device pointers unless marked host.
 *
 * goslam_neus_sdf_grid — u[i,j,k] (f32 [nx,ny,nz], z fastest) = -sdf(xs[i], ys[j], zs[k]) where the point passes the
 *   strict params->rt_bound test, -100 elsewhere; the sdf is normalised by params->bound (row 0 of the SDF head, the
 *   marcher's hash-grid gather).  xs, ys, zs are the caller's torch.linspace tables (the kernel does not recompute them).
 *
 * goslam_mc_count / goslam_mc_emit — marching cubes on u at level iso (inside iff (double)u > iso), tables generated by
 *   tools/gen_mc_tables.py.  count writes counts[0] = vertices, counts[1] = faces (device int64) and leaves its state
 *   in the workspace (goslam_mc_workspace_bytes(nx,ny,nz) bytes, 1.125 bytes per lattice point plus a little), which
 *   emit reads: call emit with the same u, shape, iso and workspace.  emit writes verts [V,3] f64 in world coordinates
 *   (the index-space position, one vertex per crossing lattice edge in ascending edge id 3*linear+axis, mapped by
 *   v / (n_axis - 1.0) * (double)(float)(bound_max - bound_min) + (double)bound_min; bound_min / bound_max are host
 *   float[3]) and faces [F,3] int64 (by cell, x-major, z fastest, then table order); it writes at most max_verts /
 *   max_faces rows.  nx, ny, nz >= 2.
 *
 * goslam_mesh_cull_count / goslam_mesh_cull_emit — keep a vertex iff lo[c] <= v[c] <= hi[c] for all c (lo, hi: host
 *   float[3], compared in f64), a face iff its three vertices are kept, then drop the vertices no kept face references;
 *   orders are stable and faces are re-indexed.  count writes counts[0] = kept vertices, counts[1] = kept faces and
 *   leaves its state in the workspace (goslam_mesh_cull_workspace_bytes) for emit, which writes at most max_out_verts /
 *   max_out_faces rows.
 *
 * goslam_neus_vertex_color — extract_color: rgb [n,3] uint8 = uint8(clip(c, 0, 1) * 255) of the colour network at the
 *   vertices rounded to f32 (normal and feature from the hash grid normalised by params->bound; no rt_bound mask).
 * ---------------------------------------------------------------------------------- */
int goslam_neus_sdf_grid(const goslam_neus_params* params, const float* xs, const float* ys, const float* zs, int nx,
                         int ny, int nz, float* u, void* stream);
size_t goslam_mc_workspace_bytes(int nx, int ny, int nz);
int goslam_mc_count(const float* u, int nx, int ny, int nz, double iso, void* workspace, size_t workspace_bytes,
                    int64_t* counts, void* stream);
int goslam_mc_emit(const float* u, int nx, int ny, int nz, double iso, const float* bound_min, const float* bound_max,
                   const void* workspace, size_t workspace_bytes, double* verts, int64_t max_verts, int64_t* faces,
                   int64_t max_faces, void* stream);
size_t goslam_mesh_cull_workspace_bytes(int64_t n_verts, int64_t n_faces);
int goslam_mesh_cull_count(const double* verts, int64_t n_verts, const int64_t* faces, int64_t n_faces, const float* lo,
                           const float* hi, void* workspace, size_t workspace_bytes, int64_t* counts, void* stream);
int goslam_mesh_cull_emit(const double* verts, int64_t n_verts, const int64_t* faces, int64_t n_faces, const void* workspace,
                          size_t workspace_bytes, double* out_verts, int64_t max_out_verts, int64_t* out_faces,
                          int64_t max_out_faces, void* stream);
int goslam_neus_vertex_color(const goslam_neus_params* params, const double* verts, int64_t n, unsigned char* rgb,
                             void* stream);
/* ------------------------------------------------------------------------------------
 * Mesh culling against the camera views: Mesher.cull_mesh (src/mesher.py:56-240).  Device pointers unless marked host.
 *
 * goslam_mesh_cull_mask_count — the count pass of goslam_mesh_cull_count with a keep rule given by masks: a face is kept
 *   iff face_mask[f] != 0 and vert_mask[v] != 0 for its three vertices (u8; either may be NULL, meaning all kept).  Fills
 *   the goslam_mesh_cull_workspace_bytes workspace for goslam_mesh_cull_emit and goslam_mesh_cull_vertex_ids, which writes
 *   the old index (int64) of every kept vertex in output order (at most max_ids) so that per-vertex attributes follow.
 *
 * goslam_mesh_depth_render — extract_depth_from_mesh: depth [K,H,W] f32 of the mesh (verts [V,3] f64, faces [F,3] i64)
 *   seen from c2w [K,4,4] f32 (OpenCV camera-to-world), pinhole fx, fy, cx, cy.  Camera coordinates R^T (p - t) in f64,
 *   clip against z = znear, pixel (r, c) samples (c + 0.5, r + 0.5), inclusive coverage of either winding, perspective-
 *   correct z, fragments with z > zfar dropped, the nearest fragment kept; 0 where no fragment lands.  K <= 65535.
 *
 * goslam_mesh_view_masks — point_masks over one chunk of views: ORs into seen[V] and forecast[V] (u8, zeroed once by the
 *   caller) with w2c [K,4,4] f32 (torch.inverse(c2w)) and depth [K,H,W] of the same views; the reference's f32 arithmetic,
 *   grid_sample bilinear / border / align_corners=True, front = d > 0 ? z < d + eps : true.
 *
 * goslam_mesh_components_count / goslam_mesh_components_keep — get_connected_mesh: faces are adjacent when they share an
 *   edge that belongs to exactly two faces; a component is kept iff its area (f64) > threshold * the mesh's area, or, with
 *   largest != 0, only the component of largest area (ties: the one with the smallest face id).  count writes counts[0] =
 *   number of components (device int64) and leaves its state in the workspace (goslam_mesh_components_workspace_bytes,
 *   which needs a device to size CUB's scratch and returns 0 without one); keep takes that number from the host and writes
 *   face_keep[F] (u8), the input of goslam_mesh_cull_mask_count.  Faces must index [0, n_verts); F < 2^31.
 * ---------------------------------------------------------------------------------- */
int goslam_mesh_cull_mask_count(int64_t n_verts, const int64_t* faces, int64_t n_faces, const unsigned char* face_mask,
                                const unsigned char* vert_mask, void* workspace, size_t workspace_bytes, int64_t* counts,
                                void* stream);
int goslam_mesh_cull_vertex_ids(int64_t n_verts, int64_t n_faces, const void* workspace, size_t workspace_bytes, int64_t* ids,
                                int64_t max_ids, void* stream);
int goslam_mesh_depth_render(const double* verts, int64_t n_verts, const int64_t* faces, int64_t n_faces, const float* c2w,
                             int K, int H, int W, double fx, double fy, double cx, double cy, double znear, double zfar,
                             float* depth, void* stream);
int goslam_mesh_view_masks(const double* verts, int64_t n_verts, const float* w2c, const float* depth, int K, int H, int W,
                           float fx, float fy, float cx, float cy, float radius, float eps, unsigned char* seen,
                           unsigned char* forecast, void* stream);
size_t goslam_mesh_components_workspace_bytes(int64_t n_verts, int64_t n_faces);
int goslam_mesh_components_count(const double* verts, int64_t n_verts, const int64_t* faces, int64_t n_faces, void* workspace,
                                 size_t workspace_bytes, int64_t* counts, void* stream);
int goslam_mesh_components_keep(int64_t n_faces, int64_t n_components, double threshold, int largest, void* workspace,
                                size_t workspace_bytes, unsigned char* face_keep, void* stream);
/* hash-grid geometry helper (host side, no GPU): fills offsets[17] (in PARAMS, i.e.
 * entries*2), resolutions[16], scales[16]; returns total number of f16 params. */
int64_t goslam_hashgrid_layout(int64_t* offsets, int* resolutions, float* scales);

/* ------------------------------------------------------------------------------------
 * Per-ray depth sampling — the z-sampling half of Renderer.render_batch_ray
 * (src/render.py:99-171: near/far from the scene AABB and the sensor depth, n_samples
 * stratified samples with one shared jitter table, n_surface samples around the sensor
 * depth, sorted union, successive distances).
 *   rays_o, rays_d [R,3] f32; bound [3,2] f32 (device); gt_depth [R] f32 or NULL (then
 *   n_surface is ignored and near = 0.01);
 *   t_samples [n_samples] = torch.linspace(0,1,n_samples); t_surface [n_surface] likewise;
 *   perturb_rand [n_samples] = torch.rand(n_samples) or NULL when rendering.perturb <= 0;
 *   z_vals, dists [R, n_samples + n_surface] f32 out.  n_samples + n_surface <= 128.
 *   workspace: >= 256 bytes (device). */
int goslam_sample_z(const float* rays_o, const float* rays_d, const float* bound,
                    const float* gt_depth, const float* t_samples, const float* t_surface,
                    const float* perturb_rand, int R, int n_samples, int n_surface, int lindisp,
                    float* z_vals, float* dists, void* workspace, size_t workspace_bytes,
                    void* stream);

/* ------------------------------------------------------------------------------------
 * Convex 8x upsampling (cvx_upsample, src/droid_net.py:9-23; DepthVideo.upsample,
 * src/depth_video.py:194-196): out[b,8y+sy,8x+sx,:] = sum_k softmax_k(mask[b,k,sy,sx,y,x]) *
 * data[b,y+ky-1,x+kx-1,:] over the zero-padded 3x3 neighbourhood, k = 3*ky + kx.
 *   data [B,ht,wd,dim] f32 (dim <= 4), mask [B,576,ht,wd] f16 or f32 (mask_dtype = GOSLAM_F16 /
 *   GOSLAM_F32; an f16 mask gives f16-rounded softmax weights, as torch.softmax does),
 *   out [B,8ht,8wd,dim] f32, fully overwritten. */
int goslam_cvx_upsample(const float* data, const void* mask, int mask_dtype, float* out, int B,
                        int ht, int wd, int dim, void* stream);

/* ------------------------------------------------------------------------------------
 * Factor-graph edge selection — FactorGraph.add_proximity_factors (src/factor_graph.py:384-450;
 * every keyframe, src/frontend.py:58) without the per-candidate device->host syncs of its Python
 * loops.  dist [(t-t0)*(t-t1)] f32 = DepthVideo.distance over the meshgrid of (t0..t-1) x (t1..t-1)
 * (goslam_frame_distance), ii_old/jj_old [n_old] = edges the graph already holds (active, bad,
 * inactive).  Writes the reference's edge list, in its order, to es_i/es_j [cap] (int64) and the
 * number of edges to *num_edges (device int).  Greedy NMS stops once more than max_factors edges
 * are listed; ties in distance are taken in index order.
 * dmax / jfloor select the variant: add_proximity_factors masks d > 100 and starts the local window
 * at max(i - rad, 0) (dmax = 100, jfloor = 0); Backend.ba without loop closure (src/backend.py:25-99)
 * masks d > thresh, starts it at max(i - radius, t_start) and holds no previous edges
 * (dmax = thresh, jfloor = t0 = t1 = t_start, n_old = 0).  loop != 0 is Backend.ba's loop-closure mode
 * (src/backend.py:81-91; t0 = t_start_loop, t1 = t_start, jfloor = t_start_loop, stereo ignored by the
 * caller): an accepted candidate contributes the cells of its 3x3 neighbourhood whose RAW distance is
 * below thresh (off-diagonal ones, row-major) when more than 4 of the 9 are.
 *   cap >= edges of the local window + max(0, max_factors + 2) (+ 8 in loop mode) is always enough.
 *   workspace: goslam_proximity_workspace_bytes(t0, t1, t). */
size_t goslam_proximity_workspace_bytes(int t0, int t1, int t);
int goslam_proximity_edges(const float* dist, int t0, int t1, int t, int rad, int nms, float thresh,
                           float dmax, int jfloor, int loop, int max_factors, int stereo,
                           const int64_t* ii_old, const int64_t* jj_old, int n_old, int64_t* es_i,
                           int64_t* es_j, int cap, int* num_edges, void* workspace,
                           size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------
 * ConvGRU of the update operator (SURVEY §8f-4).  Replaces ConvGRU.forward (src/modules/gru.py:21-39) as
 * UpdateModule calls it (src/droid_net.py:125): three wgmma implicit-GEMM convolution passes with the gate
 * arithmetic fused into their epilogues (csrc/conv_tc.cu).
 *   State and inputs are NHWC f16: net, inp, corr [B,h,w,128], flow [B,h,w,64]; net_out [B,h,w,128] (may alias
 *   nothing else).  goslam_nchw_to_nhwc_f16 / goslam_nhwc_to_nchw_f16 convert from / to the reference's
 *   [B,C,h,w] tensors ([B,C,hw] <-> [B,hw,C]).
 *   Weights (device pointers), packed from the reference module's parameters:
 *     w_zr  f16 [9][256][448]  convz.weight | convr.weight stacked along cout; tap = 3*ky + kx; cin order
 *                              net(128) | inp(128) | corr(128) | flow(64) = torch.cat order of the reference
 *     w_q   f16 [9][128][448]  convq.weight        w_w f16 [128][128]  w.weight (1x1)
 *     b_zr  f32 [256], b_q f32 [128], b_w f32 [128]
 *     w_glo f32 [384][128], b_glo f32 [384]   convz_glo | convr_glo | convq_glo (1x1 on the pooled vector)
 * ---------------------------------------------------------------------------------- */
typedef struct goslam_gru_weights {
  const void* w_zr; const void* w_q; const void* w_w;
  const float* b_zr; const float* b_q; const float* b_w;
  const float* w_glo; const float* b_glo;
} goslam_gru_weights;
size_t goslam_conv_gru_workspace_bytes(int B, int h, int w);
int goslam_conv_gru(const goslam_gru_weights* weights, const void* net, const void* inp, const void* corr,
                    const void* flow, void* net_out, int B, int h, int w, void* workspace,
                    size_t workspace_bytes, void* stream);
int goslam_nchw_to_nhwc_f16(const void* src, void* dst, int B, int C, int hw, void* stream);
/* same with the channel dimension zero-padded to Cpad (e.g. the 196 correlation channels -> 256) */
int goslam_nchw_to_nhwc_f16_pad(const void* src, void* dst, int B, int C, int Cpad, int hw, void* stream);

/* One convolution layer of the update operator (src/droid_net.py:70-105: the encoders, the delta / weight heads and
 * GraphAgg) on the same wgmma implicit-GEMM kernel: 1x1 or 3x3 (padding 1), up to four NHWC f16 inputs read as if
 * concatenated along channels (each may be a channel slice of a wider tensor), fused bias + activation.
 *   in[i]: [B,h,w,cin_stride[i]] f16, channels cin_off[i] .. cin_off[i]+cin[i] used (all multiples of 64)
 *   weight f16 [taps][cout_pad][sum cin] (tap = 3*ky + kx), bias f32 [cout_pad]; cout_pad multiple of 16 (rows
 *   cout..cout_pad-1 zero) and <= 256 or a multiple of 128 / 192 / 256; at most 1024 (the bias vector is staged in
 *   shared memory), larger layers return GOSLAM_EINVAL
 *   act: 0 none, 1 ReLU, 2 sigmoid, 3 softplus; result * out_scale
 *   out: NHWC [B,h,w,out_stride] f16 (out_f32 = 0; stride and offset multiples of 8) or f32, channels
 *   out_offset .. out_offset + cout written. */
typedef struct goslam_conv_desc {
  const void* in[4]; int cin[4]; int cin_off[4]; int cin_stride[4]; int n_in;
  const void* weight; const float* bias;
  int taps, cout, cout_pad, act;
  float out_scale;
  void* out; int out_f32, out_stride, out_offset;
  /* optional (f32 outputs, cout <= 8): channels >= split are written to out2 (same stride) as channel - split and
   * get activation act2 instead of act — two small heads in one pass over block-diagonal weights */
  int split, act2; void* out2;
} goslam_conv_desc;
int goslam_conv2d_nhwc(const goslam_conv_desc* d, int B, int h, int w, void* stream);
int goslam_nhwc_to_nchw_f16(const void* src, void* dst, int B, int C, int hw, void* stream);

/* The whole update operator in one call — UpdateModule.forward (src/droid_net.py:107-140): layout conversion of the
 * reference-shaped inputs, corr / flow encoders, ConvGRU, delta / weight heads and GraphAgg; ~20 launches issued by
 * the library on `stream`, no host synchronisation.
 *   net, inp f16 [N,128,h,w]; corr f16 [N,196,h,w] (CorrBlock.__call__'s output); flow f32 [N,4,h,w] (the motion
 *   features); frame_slot int32 [N]: index of each edge's source frame among the M distinct source frames in sorted
 *   order (GraphAgg's unique(ii, return_inverse)), or NULL to skip GraphAgg (ii is None in the reference).
 *   Outputs: net_out f16 [N,128,h,w]; delta, weight f32 [N,h,w,2]; eta f32 [M,h,w] (already times 0.01);
 *   upmask f16 [M,576,h,w].
 *   Weights (device pointers, packed like goslam_conv_desc.weight; "pad 16" = cout rows 2.. / 1.. are zero):
 *     corr0 [1][128][256] (cin 196 zero-padded), corr2 [9][128][128], flow0 f16 [128][256] with k = (ky*7+kx)*4+ci
 *     (zero beyond 196), flow2 [9][64][128], hid [9][256][128] = delta.0 | weight.0,
 *     delta_w = both 2-channel heads block-diagonal [9][16][256]: rows 0-1 delta.2 on hidden channels 0..127, rows 2-3
 *     weight.2 on 128..255, bias [16] likewise (weight_w / weight_b unused),
 *     agg1, agg2 [9][128][128], eta [9][16][128] (pad 16), upmask [1][576][128]; biases f32 [cout_pad]. */
typedef struct goslam_update_weights {
  goslam_gru_weights gru;
  const void* corr0_w; const float* corr0_b; const void* corr2_w; const float* corr2_b;
  const void* flow0_w; const float* flow0_b; const void* flow2_w; const float* flow2_b;
  const void* hid_w; const float* hid_b; const void* delta_w; const float* delta_b;
  const void* weight_w; const float* weight_b;
  const void* agg1_w; const float* agg1_b; const void* agg2_w; const float* agg2_b;
  const void* eta_w; const float* eta_b; const void* upmask_w; const float* upmask_b;
} goslam_update_weights;
size_t goslam_update_op_workspace_bytes(int N, int M, int h, int w);
int goslam_update_op(const goslam_update_weights* weights, const void* net, const void* inp, const void* corr,
                     const float* flow, const int* frame_slot, int N, int M, int h, int w, void* net_out,
                     float* delta, float* weight, float* eta, void* upmask, void* workspace,
                     size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------
 * Mapping hand-over and ray sampling: Mapper.__call__'s per-frame DepthVideo.get_mapping_item
 * (src/depth_video.py:153-173) and per-iteration build_rays (src/nerf_func.py:115-181), and render_img's
 * build_all_rays (:184-221).  Device pointers unless marked host.
 *
 * goslam_mapping_snapshot — reads the live buffers images [buffer,3,H,W], mask_filtered, disps_filtered [buffer,H,W]
 *   (f32) for the F distinct frames frames[F] (device int32) and writes, per frame f (its "slot"), the pixels whose mask
 *   value is non-zero (NaN included, as `.bool()`) as compact records in raster order: pixel id y*W + x (int32) and
 *   (r, g, b, depth) (f32) with depth = 1.0f / (disp + 1e-7f), both IEEE-rounded.  A count pass over 1024-pixel tiles,
 *   a per-frame scan of the tile counts, then an emit pass that places each tile's records at its prefix.  counts[f]
 *   (device int32) = N_f.  The same launch sequence multiplies update_priority[frames[f]] by decay occurrences[f]
 *   times (device int32), one f32-rounded multiply at a time.  Frames outside [0, buffer) give N_f = 0 and no decay.
 *   Workspace: goslam_mapping_snapshot_workspace_bytes(F, H, W) =
 *     2 * align256(4 * F * ceil(H*W / 1024)) + align256(4 * F * H*W) + align256(16 * F * H*W)
 *   (0 for F <= 0, F > 65535, H or W <= 0, or H*W > 2^26).  The records live in the workspace; nothing reads the live
 *   buffers after the three launches.
 *
 * goslam_mapping_rays — one training iteration's batch from a snapshot workspace (same F, H, W): n_entries entries
 *   (host arrays slots[], counts[] = the slot's N_f, draw[]), concatenated in entry order.  draw[e] > 0 takes draw[e]
 *   records at indices draws[...] (device int64, consecutive per entry in entry order, clamped to [0, N_f - 1]);
 *   draw[e] == 0 takes all N_f records in raster order.  Per ray, with c2w [F,4,4] (row-major f32, indexed by slot),
 *   x = column, y = row as exact floats, and from the host doubles fx..cy the f32 values cx' = (float)cx and
 *   rfx = (float)(1.0 / fx) that torch's CUDA `(x - cx) / fx` uses with Python-float intrinsics:
 *     dirs = ((x - cx') * rfx, (y - cy') * rfy, 1)
 *     rays_d[r] = (dirs.x * R[r][0] + dirs.y * R[r][1]) + R[r][2]   each product and sum rounded, no FMA
 *     rays_o = t,   depth = the record's depth,   color = the record's rgb
 *   into rays_o, rays_d, color [R,3] and depth [R] (f32), R = sum over entries of (draw > 0 ? draw : N_f) <= max_rays.
 *   Lists longer than 64 entries are launched in chunks of 64.
 *
 * goslam_mapping_all_rays — rays_o, rays_d [H*W,3] of every pixel of one image in raster order under c2w [4,4] (device),
 *   the arithmetic of goslam_mapping_rays.
 * ---------------------------------------------------------------------------------- */
size_t goslam_mapping_snapshot_workspace_bytes(int F, int H, int W);
int goslam_mapping_snapshot(const float* images, const float* mask, const float* disps, float* update_priority, int buffer,
                            int H, int W, const int* frames, const int* occurrences, int F, float decay, void* workspace,
                            size_t workspace_bytes, int* counts, void* stream);
int goslam_mapping_rays(const void* workspace, size_t workspace_bytes, int F, int H, int W, const float* c2w,
                        const int64_t* draws, int64_t n_draws, int n_entries, const int* slots, const int* counts,
                        const int* draw, double fx, double fy, double cx, double cy, float* rays_o, float* rays_d, float* depth,
                        float* color, int64_t max_rays, void* stream);
int goslam_mapping_all_rays(const float* c2w, int H, int W, double fx, double fy, double cx, double cy, float* rays_o,
                            float* rays_d, void* stream);

/* ------------------------------------------------------------------------------------
 * Feature / context encoder: DroidNet's BasicEncoder forward (src/modules/extractor.py) for norm_fn 'instance'
 * (fnet: InstanceNorm2d, biased variance, eps 1e-5, no affine) and 'none' (cnet).  Device pointers.
 *
 * Weights, one goslam_encoder_conv per nn.Conv2d: w f16 [cout][Kpad] with k = (ky * ks + kx) * cin + ci (the
 * reference's [cout][cin][ky][kx] permuted to [cout][ky][kx][cin]), Kpad = K except the stem's 147 zero-padded to 160;
 * b f32 [cout].
 *   stem        conv1, 7x7 stride 2, 3 -> 32
 *   block[i]    i = 0..5: layer1.0, layer1.1, layer2.0, layer2.1, layer3.0, layer3.1 (32, 32, 64, 64, 128, 128 out);
 *               [0] conv1 3x3 (stride 2 for i = 2, 4), [1] conv2 3x3, [2] downsample.0 1x1 stride 2 (i = 2, 4 only;
 *               ignored otherwise)
 *   out         conv2, 1x1, 128 -> out_dim
 *
 * goslam_basic_encoder — image [B,3,H,W] NCHW (f32, or f16 if image_is_f16); mean, stdv [3] f32 or both NULL: the stem
 *   reads (x - mean[c]) / stdv[c] in f32 (rounded to f16 after each op for an f16 image), then rounds to f16.
 *   out_dim % 32 == 0.  Output f16 NCHW: out [B,out_dim,H/8,W/8]; with split (out_dim == 256) out = tanh of channels
 *   0-127 and out2 = relu of channels 128-255, each [B,128,H/8,W/8], both from the f16-rounded conv output.
 *   H and W must be multiples of 8 (H*W <= 2^24), B >= 1, and with instance norm (H/8)*(W/8) > 1 (F.instance_norm
 *   rejects a 1x1 input); otherwise GOSLAM_EINVAL.  About 40 launches on `stream`, no
 *   host synchronisation; deterministic (instance statistics are merged per tile in a fixed order).
 *   Workspace: goslam_encoder_workspace_bytes(B, H, W, norm) (0 for an invalid shape or norm).
 * ---------------------------------------------------------------------------------- */
#define GOSLAM_NORM_NONE 0
#define GOSLAM_NORM_INSTANCE 1
typedef struct goslam_encoder_conv {
  const void* w; const float* b;
} goslam_encoder_conv;
typedef struct goslam_encoder_weights {
  goslam_encoder_conv stem;
  goslam_encoder_conv block[6][3];
  goslam_encoder_conv out;
} goslam_encoder_weights;
size_t goslam_encoder_workspace_bytes(int B, int H, int W, int norm);
int goslam_basic_encoder(const goslam_encoder_weights* weights, int norm, int out_dim, const void* image, int image_is_f16,
                         const float* mean, const float* stdv, int B, int H, int W, void* out, void* out2, int split,
                         void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------
 * Non-keyframe trajectory fill: PoseTrajectoryFiller.__fill's bracketing and linear SE3 interpolation
 * (src/trajectory_filler.py:38-55) and the video hand-over `video[N:N+M] = (tt, ..., Gs, 1, depths, intrinsics / 8,
 * ...)` (:62-63, src/depth_video.py:85-120), one launch on `stream` with no host synchronisation.  Device pointers.
 *
 * goslam_fill_interpolate — the video's live buffers timestamp [buffer], poses [buffer,7], intrinsics [buffer,4],
 *   disps and disps_sens [buffer,H/8,W/8] (f32), N keyframes in rows 0..N-1; the chunk's M frames: tt [M] (f32
 *   timestamps), intr_full [M,4] (full-resolution intrinsics), depth [M,H,W] (f32) or NULL.  Per frame k:
 *     t0 = (number of ts[0:N] <= tt[k]) - 1,  t1 = t0 < N-1 ? t0+1 : t0             (int64, into t0[k], t1[k])
 *     dt = ts[t1] - ts[t0] + 1e-3,  dP = P[t1] * P[t0]^-1,  v = log(dP) / dt,  w = v * (tt[k] - ts[t0]),
 *     G = exp(w) * P[t0]                                                            (f32, in this order)
 *   and row N+k receives timestamp = tt[k], poses = G, intrinsics = intr_full[k] / 8, disps = 1, and with depth
 *   disps_sens = where(d > 0, 1 / d, d) of depth[k][3::8, 3::8] and disps = disps_sens (without depth disps_sens is
 *   not written).  A frame before every keyframe (count 0) is bracketed as t0 = 0; callers reject it first.
 *   N >= 1, 0 <= M <= 65535, H and W multiples of 8; otherwise GOSLAM_EINVAL.  The caller keeps N + M <= buffer.
 * ---------------------------------------------------------------------------------- */
int goslam_fill_interpolate(float* timestamp, float* poses, float* intrinsics, float* disps, float* disps_sens, int N,
                            int M, const float* tt, const float* intr_full, const float* depth, int H, int W,
                            int64_t* t0, int64_t* t1, void* stream);

/* ------------------------------------------------------------------------------------
 * Reconstruction evaluation: align_mesh / eval_mesh (src/mesher.py:339-421): surface sampling, exact nearest-neighbour
 * search and point-to-point ICP.  Device pointers; points [n,3] f64, faces [F,3] int64.  No host synchronisation.
 *
 * goslam_mesh_sample_surface — trimesh.sample.sample_surface from caller-drawn uniforms [count,3] (u, l0, l1): face =
 *   the first f with cum[f] >= u * cum[F-1] (cum = fp64 inclusive scan of the faces' fp64 areas, a face with an index
 *   outside [0, n_verts) has area 0 and samples NaN), point = ((v1 - v0) l0 + (v2 - v0) l1) + v0 per component after
 *   (l0, l1) <- (|l0 - 1|, |l1 - 1|) when l0 + l1 > 1, every operation rounded (no FMA).  samples [count,3];
 *   face_index [count] or NULL.  Workspace: goslam_mesh_sample_workspace_bytes(n_faces); n_faces >= 1.
 *
 * goslam_nn_index_build — a uniform grid over points [n_points,3] (1 <= n_points <= 2^28, finite coordinates) built
 *   into the caller's buffer `index` (goslam_nn_index_workspace_bytes(n_points) bytes), which must stay alive and
 *   unchanged while it is queried.  Cells are at least min_cell (>= 0) wide; pass the query radius for radius queries.
 * goslam_nn_query — for each of query [n_query,3] the nearest indexed point with d2 < max_dist^2 (max_dist = +inf: no
 *   bound), d2 = (dx^2 + dy^2) + dz^2 rounded operation by operation: dist = sqrt(d2) (+inf if none) and idx = its
 *   point id (-1 if none; the smallest id among equal d2).  Exact: the result does not depend on the grid.  Either
 *   output may be NULL.
 * goslam_nn_distance_stats — out[0] = sum of dist [n], out[1] = number of dist < threshold (fixed summation order).
 *
 * goslam_icp_point_to_point — Open3D's registration_icp with TransformationEstimationPointToPoint (no scaling) of
 *   source [n_source,3] onto the indexed target: init [4,4] row-major (device, any 4x4; points are divided by w),
 *   correspondences = nearest target with d2 < threshold^2, update = Umeyama's rotation and translation of the
 *   correspondences (identity without any), T <- update T, stop after max_iteration updates or when |d fitness| <
 *   relative_fitness and |d rmse| < relative_rmse.  result [19] (device f64): T [16] row-major, fitness, inlier rmse,
 *   number of updates.  All max_iteration iterations are enqueued; kernels after convergence return at once.
 *   Workspace: goslam_icp_workspace_bytes(n_source).
 * ---------------------------------------------------------------------------------- */
size_t goslam_mesh_sample_workspace_bytes(int64_t n_faces);
int goslam_mesh_sample_surface(const double* verts, int64_t n_verts, const int64_t* faces, int64_t n_faces,
                               const double* uniforms, int64_t count, double* samples, int64_t* face_index,
                               void* workspace, size_t workspace_bytes, void* stream);
size_t goslam_nn_index_workspace_bytes(int64_t n_points);
int goslam_nn_index_build(const double* points, int64_t n_points, double min_cell, void* index, size_t index_bytes,
                          void* stream);
int goslam_nn_query(const void* index, size_t index_bytes, int64_t n_points, const double* query, int64_t n_query,
                    double max_dist, double* dist, int64_t* idx, void* stream);
int goslam_nn_distance_stats(const double* dist, int64_t n, double threshold, double* out, void* stream);
size_t goslam_icp_workspace_bytes(int64_t n_source);
int goslam_icp_point_to_point(const double* source, int64_t n_source, const void* index, size_t index_bytes,
                              int64_t n_target, double threshold, const double* init, int max_iteration,
                              double relative_fitness, double relative_rmse, double* result, void* workspace,
                              size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------
 * Scene bound of Mesher.update_param_from_mapping (src/mesher.py:242-281, src/oriented_bounding_box.py): the mapping
 * point selection, convex-hull vertices and Open3D 0.13's oriented bounding box.  Device pointers, no host
 * synchronisation.
 *
 * goslam_mapping_points_count — the multiview filter's mask1 with thresh 0.01 and visible_num 3 over the T keyframes
 *   (poses [T,7] for the votes, poses_world [T,7] = w2w * SE3(poses).inv() for the points, disps [T,ht,wd], intrinsic
 *   [4] already scaled): *count (device int64) = number of selected pixels.
 * goslam_mapping_points_emit — the selected pixels' iproj points, [b,h,w] row-major, widened to f64 [n_points,3];
 *   n_points must be the count of the preceding _count call on the same workspace.
 *   Workspace: goslam_mapping_points_workspace_bytes(T, ht, wd) (0 = invalid shape).
 *
 * goslam_hull_vertices — the vertices of the convex hull of points [n,3] f64 (1 <= n <= 2^28): the exact extreme
 *   points (a point on a hull face or edge is not one; of equal points only the lowest index can be one), sorted, kept
 *   in the workspace.  info [4] (device int64): status (0 ok, 1 fewer than four affinely independent points, 2 hull too
 *   large, 3 non-finite coordinate, 4 inconsistent facet graph), vertex count, survivors of the interior cull,
 *   distinct direction extremes.
 *   Workspace: goslam_hull_workspace_bytes(n).
 * goslam_hull_vertices_emit — the first count (= info[1]) vertex ids as int64.
 * goslam_obb_from_hull — box [15] f64 = center [3], R [9] row-major, extent [3] (+ extend) of OrientedBoundingBox::
 *   CreateFromPoints on the hull of the preceding goslam_hull_vertices call; unwritten unless its status is 0.
 * goslam_obb_in_bound — mask [n] (1 = inside) of GetPointIndicesWithinBoundingBox for the box [15] in device memory.
 * ---------------------------------------------------------------------------------- */
size_t goslam_mapping_points_workspace_bytes(int T, int ht, int wd);
int goslam_mapping_points_count(const float* poses, const float* poses_world, const float* disps,
                                const float* intrinsic, int T, int ht, int wd, void* workspace, size_t workspace_bytes,
                                int64_t* count, void* stream);
int goslam_mapping_points_emit(const float* poses_world, const float* disps, const float* intrinsic, int T, int ht,
                               int wd, void* workspace, size_t workspace_bytes, double* points, int64_t n_points,
                               void* stream);
size_t goslam_hull_workspace_bytes(int64_t n);
int goslam_hull_vertices(const double* points, int64_t n, void* workspace, size_t workspace_bytes, int64_t* info,
                         void* stream);
int goslam_hull_vertices_emit(const void* workspace, size_t workspace_bytes, int64_t n, int64_t* out, int64_t count,
                              void* stream);
int goslam_obb_from_hull(const double* points, int64_t n, const void* workspace, size_t workspace_bytes, double extend,
                         double* box, void* stream);
int goslam_obb_in_bound(const double* box, const double* points, int64_t n, uint8_t* mask, void* stream);

/* ------------------------------------------------------------------------------------
 * Trajectory evaluation of SLAM.terminate (src/slam.py:341-370): evo's APE w.r.t. the translation part with a Sim(3)
 * Umeyama alignment (main_ape.ape(..., align=True, correct_scale=True)).  Device pointers, f64, no host
 * synchronisation; the caller reads `out` once when the stream reaches it.
 *
 * goslam_ape_sim3 — est [n,3] estimated positions, ref [n,4,4] row-major reference c2w poses, 0 <= n <= 2^31 - 1.
 *   Row i is kept iff the sum of its 16 reference entries (numpy's pairwise order) is finite; kept rows stay in input
 *   order.  On the kept rows (x = est, y = ref translation): mx, my the means, sigma_x^2 = (1/n) sum |x - mx|^2,
 *   C = (1/n) sum (y - my)(x - mx)^T = U diag(d) V^T (d descending), S = diag(1, 1, det U det V < 0 ? -1 : 1),
 *   R = U S V^T, c = trace(diag(d) S) / sigma_x^2, t = my - c R mx; errors e_i = |(R (c x_i) + t) - y_i|.
 *   out [GOSLAM_APE_OUT] (device f64): status (GOSLAM_APE_*), kept rows, sim3 [16] row-major = [[c R, t], [0, 1]],
 *   the statistics rmse, mean, median (numpy's), std (population), min, max, sse, then d [3].  sim3 and the
 *   statistics are NaN unless the status is GOSLAM_APE_OK; d is NaN unless the covariance was reached.
 *   errors [n] (device f64): the kept rows' errors in input order in its first `kept` entries.  Degenerate: fewer than
 *   three kept rows, or fewer than two d_k > 2.220446049250313e-16.  Two calls on the same input give the same bits.
 *   Workspace: goslam_ape_workspace_bytes(n) (0 only for an invalid n).
 * ---------------------------------------------------------------------------------- */
#define GOSLAM_APE_OK                  0
#define GOSLAM_APE_NO_ROWS             1  /* no reference row with a finite sum      */
#define GOSLAM_APE_NONFINITE_ESTIMATE  2  /* a kept row's estimate is NaN or Inf     */
#define GOSLAM_APE_DEGENERATE          3  /* Umeyama alignment is not possible       */
#define GOSLAM_APE_STATUS    0
#define GOSLAM_APE_KEPT      1
#define GOSLAM_APE_SIM3      2
#define GOSLAM_APE_STATS    18  /* rmse, mean, median, std, min, max, sse */
#define GOSLAM_APE_SINGULAR 25
#define GOSLAM_APE_OUT      28
size_t goslam_ape_workspace_bytes(int64_t n);
int goslam_ape_sim3(const double* est, const double* ref, int64_t n, void* workspace, size_t workspace_bytes,
                    double* out, double* errors, void* stream);

/* Training-only entry points of the reference module are exported for ABI completeness
 * and return GOSLAM_EUNSUPPORTED (inference path is torch.no_grad, src/slam.py:45). */
int goslam_corr_index_backward(void);
int goslam_altcorr_backward(void);

#ifdef __cplusplus
}
#endif
#endif /* GOSLAM_B200_H_ */
