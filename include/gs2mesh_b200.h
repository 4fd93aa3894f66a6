/*
 * gs2mesh_b200 -- C ABI of the H100-native gs2mesh hot path.
 *
 * Plain C boundary (pointers + sizes, no torch / Open3D types) for the two halves of
 * the path BASELINE.json's north_star names:
 *
 *   1. forward Gaussian-splat rasterizer  -- replaces the reference's pybind seam
 *        `_C.rasterize_gaussians(...)`            DGR/ext.cpp:16, DGR/rasterize_points.h:19-39
 *        -> CudaRasterizer::Rasterizer::forward   DGR/cuda_rasterizer/rasterizer.h:30-53
 *        `_C.mark_visible(...)`                   DGR/ext.cpp:18, rasterizer.h:23-28
 *   2. TSDF voxel integration -- replaces the Open3D (0.17.0) calls the reference makes in
 *        gs2mesh_utils/tsdf_utils.py:53-56  ScalableTSDFVolume(voxel_length, sdf_trunc, RGB8)
 *        gs2mesh_utils/tsdf_utils.py:88-93  RGBDImage.create_from_color_and_depth(...)
 *        gs2mesh_utils/tsdf_utils.py:107    volume.integrate(rgbd, intrinsic, extrinsic)
 *        gs2mesh_utils/tsdf_utils.py:108    volume.extract_triangle_mesh()
 *   (DGR = third_party/gaussian-splatting/submodules/diff-gaussian-rasterization)
 *
 * Conventions
 *   - every pointer named *_dev / documented "device" is a CUDA device pointer owned by the
 *     CALLER; the library never allocates result or scratch memory (no hidden cudaMalloc on
 *     the hot path) -- query the size, allocate, pass it in;
 *   - every entry point takes the CUDA stream to enqueue on (`void*` = cudaStream_t) and never
 *     synchronises the device unless its comment says so;
 *   - return value 0 = success, anything else is a GSB_ERR_* code; gsb_last_error() gives text;
 *   - there is NO CPU fallback: without a CUDA device every compute call fails with
 *     GSB_ERR_CUDA.
 */
#ifndef GS2MESH_B200_H_
#define GS2MESH_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GSB_VERSION 100

enum {
  GSB_OK = 0,
  GSB_ERR_INVALID = 1,    /* bad argument combination (mirrors the Python Exceptions in
                             DGR/diff_gaussian_rasterization/__init__.py:191-195 and
                             AT_ERROR in rasterize_points.cu:57-59)                        */
  GSB_ERR_WORKSPACE = 2,  /* caller workspace too small; num_rendered[0] tells the need   */
  GSB_ERR_CUDA = 3,       /* CUDA runtime / launch error                                  */
  GSB_ERR_ALIGNMENT = 4   /* a device pointer is not 16-byte aligned                       */
};

const char* gsb_last_error(void);
int gsb_version(void);
/* Number of kernels this library has launched since load (bench.py's `gpu_launches`). */
uint64_t gsb_kernel_launch_count(void);

/* Optional per-stage device timing: when enabled every stage of the two pipelines is bracketed by
 * CUDA events on the launching stream.  gsb_profile_collect() synchronises the device, writes the
 * accumulated milliseconds and sample counts per stage (arrays of gsb_profile_num_stages()) and
 * resets the accumulators. */
int gsb_profile_num_stages(void);
const char* gsb_profile_stage_name(int stage);
int gsb_profile_enable(int on);
int gsb_profile_collect(double* total_ms, uint64_t* samples, int n_stages);

/* ------------------------------------------------------------------------------------------
 * Rasterizer
 * ------------------------------------------------------------------------------------------ */

/* flags for GsbRasterArgs.flags; a call with any other bit set fails with GSB_ERR_INVALID */
#define GSB_RASTER_EXACT_TILE_CULL 1u /* drop (Gaussian,tile) pairs that provably contribute to no
                                         pixel of the tile; image is bit-identical, num_rendered
                                         shrinks.  Off = reference rectangle binning
                                         (rasterizer_impl.cu:88-107).                          */
#define GSB_RASTER_NO_TMA 2u          /* stage parameters with plain loads, the path unaligned inputs
                                         always take (for tests: same results as bulk TMA)      */
#define GSB_RASTER_DEBUG_SYNC 4u      /* synchronise + check after every stage, like debug=True
                                         (auxiliary.h:166-173)                                 */
#define GSB_RASTER_CUB_SORT 8u        /* validation only: the reference's pipeline shape (P-sized scan,
                                         cub::DeviceRadixSort on tile|depth keys, host read of the
                                         instance count) instead of the in-library depth-presort +
                                         stable tile split                                      */
#define GSB_RASTER_FAST_EXP 32u       /* blend with ex2.approx in per-column / per-row exponent tables
                                         (~1e-6 relative on alpha; parity budget is 1e-4).  Off =
                                         the reference's exponent expression with full-precision
                                         expf: transmittance bit for bit the reference's        */
#define GSB_RASTER_PAIR_SHARED_DEPTH 64u /* gsb_raster_forward_pair only (left->flags): the caller asserts that both eyes see
                                         every Gaussian at the same view depth, i.e. viewmatrix[2], [6], [10], [14] are
                                         bitwise equal in the two argument blocks; ONE depth sort then serves both eyes.
                                         Verified on the device: a mismatch sets num_rendered[3].                 */
#define GSB_RASTER_ASYNC 16u          /* never wait for the stream: an undersized workspace is then
                                         reported through num_rendered[2] instead of the return
                                         value                                                 */

/* One forward rasterization.  Field-for-field the argument list of
 * CudaRasterizer::Rasterizer::forward (rasterizer.h:30-53) / RasterizeGaussiansCUDA
 * (rasterize_points.h:19-39); tensors are raw device pointers in the reference layouts. */
typedef struct GsbRasterArgs {
  int32_t P;              /* number of Gaussians                                   */
  int32_t sh_degree;      /* active SH degree D (0..3)                             */
  int32_t sh_coeffs;      /* M = coefficients stored per Gaussian (0 if shs==NULL) */
  int32_t width, height;
  const float* background;     /* device [3]                                        */
  const float* means3D;        /* device [P,3]                                      */
  const float* shs;            /* device [P,M,3] or NULL                            */
  const float* colors_precomp; /* device [P,3] or NULL   (exactly one of shs/colors) */
  const float* opacities;      /* device [P] (post-sigmoid)                         */
  const float* scales;         /* device [P,3] or NULL                              */
  const float* rotations;      /* device [P,4] (w first, normalised) or NULL        */
  const float* cov3D_precomp;  /* device [P,6] or NULL (exactly one of scales+rotations/cov3D) */
  float scale_modifier;
  const float* viewmatrix;     /* device [16]: world_view_transform as stored by cameras.py:54 */
  const float* projmatrix;     /* device [16]: full_proj_transform (cameras.py:56)   */
  const float* cam_pos;        /* device [3]                                        */
  float tan_fovx, tan_fovy;
  int32_t prefiltered;         /* accepted for signature parity; culled points never trap */
  uint32_t flags;              /* GSB_RASTER_*                                      */
  /* outputs (device).  out_color is required, the rest may be NULL. */
  float* out_color;            /* [3,H,W]                                           */
  float* out_depth;            /* [H,W]  NEW: sum_i z_i alpha_i T_i (no reference counterpart) */
  float* out_final_T;          /* [H,W]  final transmittance (ImageState.accum_alpha) */
  int32_t* radii;              /* [P]                                               */
  /* num_rendered: int64[4] written asynchronously on `stream` (device or pinned host memory);
     [0] = instances the frame bins, i.e. the instances it needs, even when that is more than
     max_instances, [1] = reference-equivalent count (sum of tile rectangles,
     what rasterize_points.cu:114 returns), [2] = 1 if the frame needed more than max_instances
     (outputs invalid), [3] = 1 if gsb_raster_forward_pair found view depths that differ between the
     eyes (outputs invalid; always 0 for gsb_raster_forward).  May be NULL.                 */
  int64_t* num_rendered;
  /* caller-owned scratch */
  void* workspace;             /* device, >= gsb_raster_workspace_bytes(...)        */
  size_t workspace_bytes;
  int64_t max_instances;       /* binning capacity the workspace was sized for      */
} GsbRasterArgs;

/* Scratch size for P Gaussians, a width x height frame and room for `max_instances`
 * (Gaussian,tile) pairs.  Replaces the three resizable byte tensors geomBuffer /
 * binningBuffer / imgBuffer of rasterize_points.cu:68-75. */
size_t gsb_raster_workspace_bytes(int32_t P, int32_t width, int32_t height, int64_t max_instances);

/* Enqueue one forward pass.  If the frame needs more than args->max_instances pairs the call
 * returns GSB_ERR_WORKSPACE (outputs are then undefined).  Without GSB_RASTER_ASYNC the call waits
 * for the stream ONCE, at the end of the frame, to be able to report that; the reference blocks in
 * the middle of the frame instead (rasterizer_impl.cu:281).  With GSB_RASTER_ASYNC nothing waits.
 * Pass num_rendered to learn how many pairs the frame needs: after GSB_ERR_WORKSPACE its [0] is
 * already written, because the call waited. */
int gsb_raster_forward(const GsbRasterArgs* args, void* stream);

/* Both eyes of a stereo pair in one call -- what Renderer.render_image_pair (renderer_utils.py:378-389) does with two
 * back-to-back forward calls on the same Gaussian cloud.  The Gaussian parameters are read ONCE (one fused preprocess
 * pass projects, bins and shades every Gaussian for both cameras).  With GSB_RASTER_PAIR_SHARED_DEPTH in left->flags the
 * Gaussians are also depth-sorted ONCE: the eyes of a rig share the camera rotation and differ by a translation along the
 * camera x axis (transformation_utils.py:219-223), so a Gaussian's view depth is the same float in both eyes whenever
 * viewmatrix[2], [6], [10], [14] are bitwise equal (about 4 of 5 rigs built like renderer_utils.py:178-206; the right
 * camera's rotation goes through a float32 Euler round trip, which moves an entry by one ulp in the others).  The kernel
 * verifies the claim: if some Gaussian's depth differs, num_rendered[3] of both eyes is set to 1 and the frames must be
 * rendered again without the flag.
 * Requirements: same P / tensors / SH settings / image size in both argument blocks, separate outputs and workspaces.
 * stream_right may be NULL (= stream_left); otherwise the right eye's binning and blending are enqueued on it, ordered
 * after the shared part by an event, so the two eyes overlap like two independent calls would.
 * Results are bit-identical to two gsb_raster_forward calls. */
int gsb_raster_forward_pair(const GsbRasterArgs* left, const GsbRasterArgs* right, void* stream_left, void* stream_right);

/* Frustum test only (rasterizer.h:23-28 markVisible): present[i] = z_view > 0.2. */
int gsb_raster_mark_visible(int32_t P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                            uint8_t* present, void* stream);

/* Post step of Renderer.render_image_pair (renderer_utils.py:389-390) on the GPU:
 * CHW float [0,1] -> HWC uint8 with cv2's saturate_cast<uchar>(x*255) (round-half-even). */
int gsb_image_to_u8(const float* chw, int32_t width, int32_t height, uint8_t* hwc, void* stream);

/* ------------------------------------------------------------------------------------------
 * TSDF volume
 * ------------------------------------------------------------------------------------------ */

#define GSB_BRICK 16               /* Open3D volume_unit_resolution default               */
#define GSB_BRICK_VOXELS 4096

/* Open3D's ScalableTSDFVolume on the GPU: an UNBOUNDED set of bricks (= Open3D "volume units", 16^3 voxels,
 * unit_length = 16*voxel_length) addressed by their integer lattice index (bx,by,bz) through a device hash table and
 * stored in a brick pool, opened on first touch like Open3D's unordered_map<Vector3i, VolumeUnit>
 * (tsdf_utils.py:53-56: no origin, no extent).  Voxel (bx,by,bz | x,y,z) has its centre at
 *     (brick_index * 16 + xyz + 0.5) * voxel_length
 * i.e. exactly on Open3D's lattice; inside a brick voxels sit at x*256 + y*16 + z (UniformTSDFVolume::IndexOf).
 * All arrays are caller-allocated device memory (the library never allocates):
 *   tsdf_weight / color / brick_index / hash_vals / hash_stamp / brick_list / counters zero-initialised,
 *   hash_keys initialised to all-ones bytes (0xFF).
 * Lattice indices must lie in [-2^20, 2^20) per axis: cells of a brick box outside that range are never stored and are
 * counted apart from pool drops (counters[2] / [6]), since a larger pool cannot hold them.  When the pool is exhausted
 * further bricks are dropped and counted (counters[1] / [5], gsb_tsdf_last_stats); the caller grows the pool and
 * integrates again. */
typedef struct GsbVolumeDesc {
  double voxel_length;
  double sdf_trunc;
  uint32_t pool_bricks;    /* capacity of the brick pool                                              */
  uint32_t hash_slots;     /* power of two >= 2 * pool_bricks                                         */
  float* tsdf_weight;      /* device [pool_bricks*4096*2]  (tsdf, weight) interleaved, per pool slot   */
  float* color;            /* device [pool_bricks*4096*4]  (r,g,b,unused) running mean, or NULL        */
  int32_t* brick_index;    /* device [pool_bricks*4]   lattice index (bx,by,bz,0) of every pool slot   */
  uint64_t* hash_keys;     /* device [hash_slots]      packed lattice index, all-ones = empty          */
  uint32_t* hash_vals;     /* device [hash_slots]      pool slot of the entry                          */
  uint32_t* hash_stamp;    /* device [hash_slots]      last frame id that queued the entry             */
  uint32_t* brick_list;    /* device [hash_slots]      scratch: entries touched by the current frame   */
  uint32_t* counters;      /* device [8]  [0] entries queued this frame, [1] bricks dropped this frame,
                                          [2] brick-box cells outside the lattice this frame,
                                          [4] pool slots in use, [5] bricks dropped since creation,
                                          [6] brick-box cells outside the lattice since creation       */
} GsbVolumeDesc;

typedef struct GsbVolume GsbVolume; /* opaque; owns no device memory */

GsbVolume* gsb_tsdf_create(const GsbVolumeDesc* desc);
void gsb_tsdf_destroy(GsbVolume* vol);

/* Per-view depth preparation, fused T0/T0b (tsdf_utils.py:78-93 + Open3D ConvertDepthToFloatImage):
 *   d = depth_in;                       (if alpha != NULL: d = alpha > alpha_min ? d / alpha : 0
 *                                        -- expected depth from the rasterizer's sum z*alpha*T)
 *   if (mask != NULL) d *= mask;        (object / occlusion masks, uint8 0/1)
 *   if (d < min_depth) d = 0;           (tsdf_utils.py:83)
 *   d /= (float)depth_scale; if ((double)d >= depth_trunc) d = 0;   (T0b)
 * final_T is the rasterizer's transmittance (alpha = 1 - final_T) or NULL. */
int gsb_tsdf_prepare_depth(const float* depth_in, const float* final_T, const uint8_t* mask, int32_t width, int32_t height,
                           float alpha_min, float min_depth, double depth_scale, double depth_trunc, float* depth_out,
                           void* stream);

/* T0 mask filters (tsdf_utils.py:73-77: cv2.morphologyEx(mask, MORPH_CLOSE, ones(k,k)) = dilate then erode, and
 * cv2.erode(mask, ones(k,k))): one k x k rectangular max (dilate != 0) or min filter over a uint8 [H,W] device mask with
 * OpenCV's window (anchor k/2; pixels outside the image ignored). kernel_size in 1..64; out must not alias in. */
int gsb_mask_morphology(const uint8_t* mask_in, int32_t width, int32_t height, int32_t kernel_size, int32_t dilate,
                        uint8_t* mask_out, void* stream);

/* Largest frame gsb_tsdf_integrate / gsb_tsdf_touch accept (larger ones fail with GSB_ERR_INVALID): the voxel update
 * packs the pixel it samples as (v << 16) | u in one int. */
#define GSB_TSDF_MAX_WIDTH 65536
#define GSB_TSDF_MAX_HEIGHT 32768

/* volume.integrate(rgbd, intrinsic, extrinsic): depth = prepared float depth [H,W] (device),
 * rgb = uint8 [H,W,3] (device) or NULL, extrinsic_w2c = row-major double[16] on the HOST
 * (what tsdf_utils.py:107 passes: inv(left_camera['extrinsic'])).  width <= GSB_TSDF_MAX_WIDTH,
 * height <= GSB_TSDF_MAX_HEIGHT. */
int gsb_tsdf_integrate(GsbVolume* vol, const float* depth, const uint8_t* rgb, int32_t width, int32_t height, double fx,
                       double fy, double cx, double cy, const double* extrinsic_w2c, void* stream);

/* Block discovery only (T1): opens the bricks the frame would touch without updating any voxel.  Lets a caller that must
 * never lose a brick (the Open3D-shaped facade) check gsb_tsdf_last_stats and grow the pool BEFORE integrating. */
int gsb_tsdf_touch(GsbVolume* vol, const float* depth, int32_t width, int32_t height, double fx, double fy, double cx, double cy,
                   const double* extrinsic_w2c, void* stream);

/* (mean, weight) -> (sum, weight) / back, in place, of every pool slot in use: (tsdf*w, w, rgb*w) / (tsdf/w, w, rgb/w).
 * The cross-rank merge below converts with the same arithmetic. */
int gsb_tsdf_to_sums(GsbVolume* vol, void* stream);
int gsb_tsdf_from_sums(GsbVolume* vol, void* stream);

/* Lattice indices (device int32[n*4]: bx,by,bz,unused) -> pool slots (device uint32[n]; 0xFFFFFFFF = not in the volume).
 * insert != 0 opens missing bricks (zero-filled) like a touch by integrate would.  `scratch` = device uint32[n]. */
int gsb_tsdf_find_bricks(GsbVolume* vol, const int32_t* indices, uint32_t n, int insert, uint32_t* slots, uint32_t* scratch,
                         void* stream);

/* A window of the lattice (bricks brick_origin + [0, brick_count) per axis, host int32[3] each) as dense x*NY*NZ + y*NZ + z
 * grids with dims = brick_count*16, for consumers that want Open3D UniformTSDFVolume indexing; bricks that were never
 * opened read as (0, 0).  tsdf / weight: device float [nx*ny*nz], either may be NULL. */
int gsb_tsdf_export_dense(const GsbVolume* vol, const int32_t* brick_origin, const int32_t* brick_count, float* tsdf,
                          float* weight, void* stream);

/* Statistics, read back asynchronously into `out` (device or pinned host, uint32[8]): [0] bricks touched by the last
 * integrate, [1] bricks it had to drop (pool exhausted, including keys left without a slot by an earlier overflow),
 * [2] frame id, [3] pool slots in use, [4] bricks dropped since creation, [5] brick-box cells of the last integrate outside
 * the lattice range [-2^20, 2^20) (one per sampled pixel and cell, not de-duplicated), [6] the same since creation.
 * gsb_tsdf_find_bricks with insert != 0 adds its drops and out-of-range indices to the same words. */
int gsb_tsdf_last_stats(const GsbVolume* vol, uint32_t* out, void* stream);

/* ------------------------------------------------------------------------------------------
 * Multi-GPU merge of view-sharded volumes (SURVEY.md 8(b) seam 2, 8(e)): ONE call per rank,
 *     gsb_tsdf_reduce(vol, comm, nranks, rank, root, scratch, scratch_bytes, &required_bytes, stream)
 * enqueues, on `stream`,
 *   1. an ncclAllGather of every rank's brick lattice indices (fixed-size message, no host round trip),
 *   2. the insertion of the other ranks' bricks into this rank's hash (the receiving ranks open them zero-filled),
 *   3. an ncclBroadcast of the root's brick order (the canonical order of the exchange),
 *   4. one fused pack kernel: (mean,w) -> (sum,w) of every brick, gathered in canonical order into `scratch`,
 *   5. ONE ncclReduce (root >= 0) / ncclAllReduce (root < 0) of the packed buffer,
 *   6. one fused unpack kernel on the receiving rank(s): (sum,w) -> (mean,w) back into the pool.
 * The only host synchronisation is the read of one 32-bit word (the size of the union, which NCCL needs as a count).
 * `comm` is an ncclComm_t (from gsb_comm_create or any other owner); NCCL is resolved from the process at run time
 * (the libnccl.so.2 torch already loaded), the library does not link against it.
 * scratch: device, >= gsb_tsdf_reduce_scratch_bytes(vol, nranks, bricks in the union) bytes. */
size_t gsb_tsdf_reduce_scratch_bytes(const GsbVolume* vol, int nranks, uint32_t union_bricks);
/* Returns GSB_ERR_WORKSPACE when `scratch` cannot hold the packed union (known only after the index exchange); it has then
 * written the size to retry with to *required_bytes (host; may be NULL).  The required size is the same on every rank, so
 * ranks that pass equally sized scratch blocks take the same decision (a collective must not be entered by some ranks
 * only); a retry repeats the cheap index exchange.  root >= 0: ncclReduce to `root` (only its volume is changed);
 * root < 0: ncclAllReduce (every rank ends with the merged volume).  Bricks a receiving rank's pool cannot hold are
 * dropped and counted like an integrate's (counters[1] / [5]).
 * Precondition: every rank passes a volume with the same pool_bricks and the same colour setting (colour on every rank or
 * on none), and the same scratch_bytes; the element counts of the collectives are derived from them, so ranks that differ
 * enter mismatched collectives.  TSDFVolume.reduce_across_ranks agrees on them before the call.
 * A GSB_ERR_WORKSPACE returned after the index exchange (scratch holds the fixed part but not the payload) leaves the
 * union's bricks opened, zero-filled, on the receiving ranks; a retry finds them and gives the bits a first call with
 * enough scratch gives. */
int gsb_tsdf_reduce(GsbVolume* vol, void* nccl_comm, int nranks, int rank, int root, void* scratch, size_t scratch_bytes,
                    size_t* required_bytes, void* stream);
/* Communicator helpers (thin wrappers of ncclGetUniqueId / ncclCommInitRank / ncclCommDestroy): rank 0 creates the
 * 128-byte id, distributes it by any means (torch.distributed broadcast in gs2mesh_b200/tsdf.py), every rank calls
 * gsb_comm_create with it; returns the ncclComm_t as an opaque pointer (NULL on failure, see gsb_last_error). */
int gsb_comm_unique_id(void* id128);
void* gsb_comm_create(const void* id128, int nranks, int rank);
void gsb_comm_destroy(void* nccl_comm);

/* ------------------------------------------------------------------------------------------
 * Mesh extraction: volume.extract_triangle_mesh() + compute_vertex_normals()
 * (gs2mesh_utils/tsdf_utils.py:108-110; Open3D ScalableTSDFVolume::ExtractTriangleMesh)
 * ------------------------------------------------------------------------------------------
 * Marching cubes over the pool slots listed in `bricks` (device uint32[n_bricks], normally every slot in use).
 * A cube is skipped when any of its 8 corners has weight 0 (corners in bricks that were never opened count as
 * weight 0, like Open3D's hash-map miss); corners are inside when tsdf < 0.  Vertices are identified by an edge
 * key = ((gx*NY + gy)*NZ + gz)*3 + axis over the voxel grid of `window` (host int32[6]: brick origin, brick count of a
 * box containing every listed brick and its +1 neighbours, e.g. the bounding box of the pool + 1); the caller
 * sorts/uniques the keys (that is the de-duplication Open3D does with a hash map) and asks for the attributes of the
 * unique edges.  The keys must fit 63 bits: 16^3 * nbx * nby * nbz * 3 < 9e18, otherwise GSB_ERR_INVALID.
 *   gsb_mesh_count    tri_counts[b]  = triangles produced by brick b
 *   gsb_mesh_emit     edge_keys[3*t..3*t+2] for every triangle, brick b writing from tri_offsets[b]
 *   gsb_mesh_vertices xyz and rgb in [0,1] (or NULL) of n unique keys, fp64 [n,3] each, equal to Open3D's doubles
 *                     (one rounding per operation in Open3D's order)
 *   gsb_mesh_vertex_normals TriangleMesh::ComputeVertexNormals() (fp64 [n_vertices,3]) of an indexed mesh, deterministic.
 *                     The caller passes the vertex -> triangle incidence as CSR: incidence = the positions 3*t+k of
 *                     triangles[] sorted by vertex id, ties in ascending position (a stable sort of the flattened
 *                     array), incidence_offsets[n_vertices + 1] = where each vertex's run starts. */
int gsb_mesh_count(const GsbVolume* vol, const int32_t* window, const uint32_t* bricks, uint32_t n_bricks, uint32_t* tri_counts,
                   void* stream);
int gsb_mesh_emit(const GsbVolume* vol, const int32_t* window, const uint32_t* bricks, uint32_t n_bricks, const int64_t* tri_offsets,
                  int64_t* edge_keys, void* stream);
int gsb_mesh_vertices(const GsbVolume* vol, const int32_t* window, const int64_t* keys, int64_t n, double* xyz, double* rgb,
                      void* stream);
int gsb_mesh_vertex_normals(const double* xyz, int64_t n_vertices, const int64_t* triangles, int64_t n_triangles,
                            const int64_t* incidence, const int64_t* incidence_offsets, double* normals, void* stream);

/* Cluster cleaning (gs2mesh_utils/tsdf_utils.py:122-142: TriangleMesh::ClusterConnectedTriangles, removal of the
 * triangles of small clusters, remove_unreferenced_vertices).  triangles: device int64 [n_triangles,3], every index in
 * [0, n_vertices) (not checked on the device).  n_triangles and n_vertices <= 2^31 - 1 (ids are 32-bit), otherwise
 * GSB_ERR_INVALID.  Both entries use one caller workspace of gsb_mesh_cluster_workspace_bytes() (0 for invalid sizes).
 *   gsb_mesh_clusters  triangles sharing an edge (either orientation; a degenerate edge (a,a) counts, a shared vertex
 *                      does not) form a cluster.  labels[t]: device int64 [n_triangles], clusters numbered in the order
 *                      of their smallest triangle (Open3D's and scipy's numbering); counts: device int64 [n_triangles],
 *                      triangles per cluster in [0, *n_clusters); n_clusters: device int64.  cluster_area (device double
 *                      [n_triangles], or NULL to skip; needs vertices = device double [n_vertices,3]): the sum of
 *                      0.5*||(v1-v0) x (v2-v0)|| over each cluster, per triangle with numpy's roundings, summed in a
 *                      fixed order (the same bits on every run, not numpy's sequential sum).
 *   gsb_mesh_remove_small_clusters  given labels / counts of gsb_mesh_clusters: keeps triangle t iff
 *                      !(counts[labels[t]] < threshold), in order, then the referenced vertices, in order.
 *                      out_triangles: device int64 [n_triangles,3] (the kept triangles with new vertex ids);
 *                      vertex_ids: device int64 [n_vertices] (old id of each kept vertex); sizes: device int64 [2] =
 *                      (kept triangles, kept vertices). */
size_t gsb_mesh_cluster_workspace_bytes(int64_t n_triangles, int64_t n_vertices);
int gsb_mesh_clusters(const int64_t* triangles, int64_t n_triangles, int64_t n_vertices, const double* vertices, void* workspace,
                      size_t workspace_bytes, int64_t* labels, int64_t* counts, int64_t* n_clusters, double* cluster_area,
                      void* stream);
int gsb_mesh_remove_small_clusters(const int64_t* triangles, int64_t n_triangles, int64_t n_vertices, const int64_t* labels,
                                   const int64_t* counts, double threshold, void* workspace, size_t workspace_bytes,
                                   int64_t* out_triangles, int64_t* vertex_ids, int64_t* sizes, void* stream);

/* ------------------------------------------------------------------------------------------
 * Mesh-quality evaluation (evaluation/DTU/eval_code/eval.py, MobileBrick evaluate.py) without Open3D / sklearn.
 * All arithmetic is fp64 with explicit roundings (no FMA contraction), in the reference's operation order.
 * ------------------------------------------------------------------------------------------
 * Surface sampling (eval.py:48-71), two passes:
 *   gsb_eval_sample_count  tri_counts[t] = points triangle t contributes (0 for zero-area triangles)
 *   gsb_eval_sample_emit   writes them (fp64 xyz) at samples + 3*tri_offsets[t], in np.mgrid order
 * vertices: device double [n_vertices,3]; triangles: device int64 [n_triangles,3]; thresh = downsample_density. */
int gsb_eval_sample_count(const double* vertices, int64_t n_vertices, const int64_t* triangles, int64_t n_triangles, double thresh,
                          int64_t* tri_counts, void* stream);
int gsb_eval_sample_emit(const double* vertices, int64_t n_vertices, const int64_t* triangles, int64_t n_triangles, double thresh,
                         const int64_t* tri_offsets, double* samples, void* stream);

/* Uniform grid over reference points: point ids counting-sorted by cell (x-major, cell index (cx*dims[1]+cy)*dims[2]+cz,
 * cx = floor((x - origin[0]) / cell)).  origin / dims must cover every point: a point outside would be clamped into a
 * border cell, and the searches below are only exact when each point lies in its cell. */
typedef struct GsbPointGrid {
  double origin[3];
  double cell;              /* cell edge length, > 0                                   */
  int32_t dims[3];          /* cells per axis, each <= 2^21; dims[0]*dims[1]*dims[2] < 2^31 */
  const double* points;     /* device double [n_points,3]                             */
  int64_t n_points;
  int64_t* cell_start;      /* device int64 [cells+1]: ids of cell c are ids[cell_start[c] .. cell_start[c+1]) */
  int64_t* ids;             /* device int64 [n_points]                                */
} GsbPointGrid;

size_t gsb_eval_grid_workspace_bytes(int64_t n_points, int64_t n_cells);
/* Fills grid->cell_start and grid->ids (order inside a cell is unspecified). */
int gsb_eval_grid_build(const GsbPointGrid* grid, void* workspace, size_t workspace_bytes, void* stream);
/* Exact 1-nearest neighbour of every query among the grid's points: dist = sqrt(((dx*dx)+dy*dy)+dz*dz) (sklearn's kd_tree
 * kneighbors distance, bit for bit), index = the nearest point (lowest index among equal squared distances).  Queries
 * with no point closer than max_dist get dist = +inf, index = -1, and the search stops there; max_dist = +inf searches
 * until the nearest point is found.  A query with a NaN or infinite coordinate gets dist = +inf, index = -1 without a
 * search.  Grids with more than 2^21 cells on an axis are refused (GSB_ERR_INVALID) by every gsb_eval_* grid call. */
int gsb_eval_nearest(const GsbPointGrid* grid, const double* queries, int64_t n_queries, double max_dist, double* dist,
                     int64_t* index, void* stream);
/* Greedy radius downsampling of the grid's points in index order (eval.py:88-93): keep[p] = 1 iff no earlier kept point q
 * has ((dx*dx)+dy*dy)+dz*dz <= radius*radius (sklearn radius_neighbors, inclusive).  Needs grid->cell > radius.
 * Runs rounds of the parallel greedy rule and reads the undecided count every 4 rounds: SYNCHRONISES the stream.
 * keep: device uint8[n_points]; counters: device uint32[4] scratch; host_undecided: pinned host uint32[1];
 * rounds (may be NULL) receives the number of rounds run. */
int gsb_eval_radius_downsample(const GsbPointGrid* grid, double radius, uint8_t* keep, uint32_t* counters,
                               uint32_t* host_undecided, int32_t* rounds, void* stream);

/* k nearest neighbours and normal estimation on the grid (gsb_normals.cu).  k is at most GSB_KNN_MAX_K: each thread
 * keeps its k best candidates in local memory.  Calls with k outside 1..GSB_KNN_MAX_K, a negative count or a missing
 * pointer are refused (GSB_ERR_INVALID) before anything is enqueued.
 *   gsb_eval_knn               the k nearest grid points of each query, exact: row i of dist2 / index (device double /
 *                              int64 [n_queries, k]) holds ((dx*dx)+dy*dy)+dz*dz and the point's index in ascending
 *                              (dist2, index) order, so among equal squared distances the lower index comes first, at
 *                              the k-th place too.  Rows of grids with fewer than k points end in (+inf, -1); a query
 *                              with a NaN or infinite coordinate gets only (+inf, -1).
 *   gsb_eval_estimate_normals  Open3D 0.17 PointCloud::EstimateNormals(KDTreeSearchParamKNN(k)) with
 *                              fast_normal_computation, for a cloud without normals: per point (device double [n,3]),
 *                              the covariance of its gsb_eval_knn neighbours (the point itself included when it is a
 *                              grid point; the identity for fewer than 3), the eigenvector of its smallest eigenvalue by
 *                              FastEigen3x3, and (0, 0, 1) where that is zero.  No orientation.  normals: device double
 *                              [n,3].  DESIGN.md section 7d gives the operation order. */
#define GSB_KNN_MAX_K 32
int gsb_eval_knn(const GsbPointGrid* grid, const double* queries, int64_t n_queries, int32_t k, double* dist2,
                 int64_t* index, void* stream);
int gsb_eval_estimate_normals(const GsbPointGrid* grid, const double* points, int64_t n_points, int32_t k, double* normals,
                              void* stream);

/* Tanks and Temples evaluation (evaluation/TNT/eval_code/python_toolbox/evaluation), restating Open3D 0.17's
 * PointCloud::Transform, SelectionPolygonVolume::CropInPolygon, VoxelDownSample and RegistrationICP with
 * TransformationEstimationPointToPoint (Eigen::umeyama); DESIGN.md section 7d gives each operation order.
 *   gsb_eval_transform_points  out[i] = (T (p_i, 1)).xyz / (T (p_i, 1)).w, rows ((T_r0*x + T_r1*y) + T_r2*z) + T_r3.
 *                              transform: host double [4][4] row-major.  out may equal points.
 *   gsb_eval_crop_polygon      keep[i] = 1 iff axis_min <= p_w <= axis_max and p lies inside the polygon (odd count of edge
 *                              crossings below p_u); orthogonal_axis 0/1/2 = x/y/z picks (u, v, w) = (1,2,0)/(0,2,1)/(0,1,2).
 *                              polygon: device double [n_vertices,3], 3 <= n_vertices <= GSB_EVAL_MAX_POLYGON.
 *                              counter: device uint32 scratch; host_non_finite: pinned host uint32.  SYNCHRONISES the
 *                              stream and returns GSB_ERR_INVALID when a point is not finite.
 *   gsb_eval_voxel_downsample  the mean of the points of each voxel floor((p - lo) / voxel_size), lo = min_bound -
 *                              voxel_size/2, summed in input order, one output point per voxel in ascending (x, y, z)
 *                              voxel order.  min_bound / max_bound: host double [3], the points' bounds.  out: device
 *                              double [n_points,3]; n_out: device int64, the number of voxels.  GSB_ERR_INVALID when
 *                              voxel_size * INT_MAX < the padded extent (Open3D's "voxel_size is too small") or when the
 *                              voxel keys need more than 63 bits.  n_points < 2^31.
 *   gsb_eval_icp_correspond    index[i] = the nearest grid point with ((dx*dx)+dy*dy)+dz*dz < radius*radius, else -1;
 *                              dist2[i] its squared distance (+inf for -1).  A source point with a NaN or infinite
 *                              coordinate gets -1.
 *   gsb_eval_icp_moments       sums over the correspondences (index[i] >= 0) with a fixed reduction tree (the same bits on
 *                              every run): pass 0 writes out[0..6] = (sum dist2, sum source xyz, sum target[index] xyz);
 *                              pass 1, given means = host double [6] (source mean, target mean), writes out[0..8] =
 *                              sum (t - mu_t)_j (s - mu_s)_k (j-major) and out[9..11] = sum (s - mu_s)_k^2.  out[12] =
 *                              the number of correspondences.  out: device double [13]; workspace: device double
 *                              [GSB_EVAL_ICP_MOMENT_WORKSPACE]. */
#define GSB_EVAL_MAX_POLYGON 2048
#define GSB_EVAL_ICP_MOMENT_WORKSPACE (13 * 256)
int gsb_eval_transform_points(const double* points, int64_t n_points, const double* transform, double* out, void* stream);
int gsb_eval_crop_polygon(const double* points, int64_t n_points, const double* polygon, int32_t n_vertices,
                          int32_t orthogonal_axis, double axis_min, double axis_max, uint8_t* keep, uint32_t* counter,
                          uint32_t* host_non_finite, void* stream);
size_t gsb_eval_voxel_workspace_bytes(int64_t n_points);
int gsb_eval_voxel_downsample(const double* points, int64_t n_points, const double* min_bound, const double* max_bound,
                              double voxel_size, void* workspace, size_t workspace_bytes, double* out, int64_t* n_out,
                              void* stream);
int gsb_eval_icp_correspond(const GsbPointGrid* grid, const double* source, int64_t n_source, double radius, int64_t* index,
                            double* dist2, void* stream);
int gsb_eval_icp_moments(const double* source, const int64_t* index, const double* dist2, int64_t n_source,
                         const double* target, int pass, const double* means, double* workspace, double* out, void* stream);

/* Mesh culling by object masks (evaluation/DTU/eval_code/evaluate_single_scene.py:21-116, `cull_scan`).
 * Binary dilation of n_views masks (device uint8 [n_views,height,width], nonzero = set) by the disk x*x + y*y <= r*r
 * (skimage disk(r)); pixels outside the image are unset.  packed: device uint32 [n_views][height][(width+31)/32], pixel x
 * of a row is bit x%32 of word x/32.  workspace: device uint8 [n_views*height*width].  0 <= radius <= 254. */
int gsb_eval_mask_dilate_disk(const uint8_t* masks, int32_t n_views, int32_t height, int32_t width, int32_t radius,
                              uint32_t* packed, uint8_t* workspace, void* stream);
/* keep[i] = 0 iff some view projects vertex i (device double [n_vertices,3], rounded to fp32) strictly inside the
 * image_width x image_height frame onto an unset pixel of its packed mask (mask_width x mask_height, the layout of
 * gsb_eval_mask_dilate_disk), else 1.  matrices: device float [n_views][4][4], row-major, camera = M @ (x, y, z, 1).
 * fp32 arithmetic in the reference's torch order on the GPU (DESIGN.md section 7a); no test of depth > 0, and a
 * non-finite projection is never culled. */
int gsb_eval_cull_vertices_by_masks(const double* vertices, int64_t n_vertices, const float* matrices, int32_t n_views,
                                    int32_t image_width, int32_t image_height, int32_t mask_width, int32_t mask_height,
                                    const uint32_t* packed_masks, uint8_t* keep, void* stream);

/* MobileBrick evaluation (evaluation/MobileBrick/eval_code/evaluate.py:34-108), restating Open3D 0.17's
 * TriangleMesh::GetSurfaceArea, SamplePointsUniformlyImpl and SamplePointsPoissonDisk and the reference's grid_sample
 * visibility test; DESIGN.md section 7e gives each operation order.  vertices: device double [n_vertices,3]; triangles:
 * device int64 [n_triangles,3].
 *   gsb_eval_triangle_areas     areas[t] = 0.5 * |(p0 - p1) x (p0 - p2)|, the norm as sqrt((x*x + y*y) + z*z).
 *   gsb_eval_sample_uniform     sample j of n_samples lies on the triangle t with bounds[t] <= j < bounds[t+1] (bounds:
 *                               device int64 [n_triangles+1], nondecreasing, bounds[0] = 0); with r1 = variates[2j],
 *                               r2 = variates[2j+1] (device double [2*n_samples]), a = 1 - sqrt(r1), b = sqrt(r1)*(1 - r2),
 *                               c = sqrt(r1)*r2, samples[j] = (a*p0 + b*p1) + c*p2.  Samples j >= bounds[n_triangles] are
 *                               (0,0,0).  n_triangles >= 1.
 *   gsb_eval_poisson_neighbours the radius neighbours of each grid point p: every q != p with ((dx*dx)+dy*dy)+dz*dz <
 *                               r_max*r_max (dx = p.x - q.x).  Needs grid->cell > r_max and fewer than 2^31 points.  With
 *                               offsets NULL it writes counts[p] (device int64 [n_points]); with offsets (device int64
 *                               [n_points+1], the exclusive scan of the counts and the total) it writes each list at
 *                               neighbours + offsets[p] (device int32), sorted by (squared distance, index), and terms[k]
 *                               = (1 - max(sqrt(d2), r_min)/r_max)^8, the power as three squarings (device double).
 *                               The emit call reads offsets[n_points] back: it SYNCHRONISES the stream.
 *   gsb_eval_poisson_eliminate  weighted sample elimination as rounds: a point's weight is the sum of its live neighbours'
 *                               terms in list order; each round deletes every live point whose key (weight, index) exceeds
 *                               the keys of all its live neighbours.  Runs until every point is deleted: weight (device
 *                               double [n_points]) then holds each point's removal key, round_of (device int32 [n_points])
 *                               the round that deleted it (from 1).  Open3D's loop keeps the number_of_points points of
 *                               smallest (weight, index).  Reads the live count every 4 rounds: SYNCHRONISES the stream.
 *                               counters: device uint32[4] scratch; host_live: pinned host uint32[4]; rounds (may be NULL)
 *                               receives the number of rounds.
 *   gsb_eval_visibility         keep[i] = 1 iff grid_sample(volume, g, nearest, zeros, align_corners=True) > 0 for
 *                               g = fp32(((((p - min_pts)/voxel_size) / (res - 1)) * 2) - 1) (fp64 until the rounding), axes
 *                               reordered to (z, y, x); volume: device uint8 [res0][res1][res2], nonzero where the
 *                               reference's float volume is > 0.  min_pts: host double [3]; resolution: host int32 [3], each
 *                               >= 2. */
int gsb_eval_triangle_areas(const double* vertices, int64_t n_vertices, const int64_t* triangles, int64_t n_triangles,
                            double* areas, void* stream);
int gsb_eval_sample_uniform(const double* vertices, int64_t n_vertices, const int64_t* triangles, int64_t n_triangles,
                            const int64_t* bounds, const double* variates, int64_t n_samples, double* samples, void* stream);
int gsb_eval_poisson_neighbours(const GsbPointGrid* grid, double r_max, double r_min, int64_t* counts,
                                const int64_t* offsets, int32_t* neighbours, double* terms, void* stream);
int gsb_eval_poisson_eliminate(const int64_t* offsets, const int32_t* neighbours, const double* terms, int64_t n_points,
                               double* weight, int32_t* round_of, uint32_t* counters, uint32_t* host_live, int32_t* rounds,
                               void* stream);
int gsb_eval_visibility(const double* vertices, int64_t n_vertices, const double* min_pts, double voxel_size,
                        const int32_t* resolution, const uint8_t* volume, uint8_t* keep, void* stream);

/* ------------------------------------------------------------------------------------------
 * Stereo stage (gs2mesh_utils/stereo_utils.py:82-179) around the caller's disparity model.
 * ------------------------------------------------------------------------------------------
 * Frames are width x height with 1 <= width <= GSB_TSDF_MAX_WIDTH, 1 <= height <= GSB_TSDF_MAX_HEIGHT.  The model's
 * inputs are padded like DLNR's InputPadder(dims, divis_by=32) ('sintel'): ph = ((H/32 + 1)*32 - H) % 32 (pw likewise),
 * [l, r, t, b] = [pw/2, pw - pw/2, ph/2, ph - ph/2], Hp = H + t + b, Wp = W + l + r.
 *   gsb_stereo_pack_inputs      left / right: device uint8 [H,W,3]; out: device float [4,3,Hp,Wp] =
 *                               pad(left), pad(right), flip_x(pad(right)), flip_x(pad(left)), replicate padding, float(u8).
 *   gsb_stereo_disparities      flow_lr / flow_rl: the model's full-resolution outputs, device float [Hp,Wp];
 *                               disp_lr[y][x] = sign * flow_lr[t+y][l+x] (device float [H,W]),
 *                               disp_rl[y][x] = sign * flow_rl[y][Wp-1-x] (device float [Hp,Wp], not cropped).
 *                               Outputs must not alias the inputs.
 *   gsb_stereo_occlusion_depth  get_occlusion_mask(disp_lr, disp_rl, threshold) and depth = fx*B / disp_lr per pixel, in
 *                               numpy's dtypes (DESIGN.md section 7c): visible (device uint8 [H,W], 1 = visible) reads row y,
 *                               column xc of disp_rl with row stride rl_stride >= width (elements); depth (device float
 *                               [H,W]) = depth_numerator / disp_lr in fp32, depth_numerator = float(fx * B) rounded once on
 *                               the host.  Either output may be NULL (not both); disp_rl may be NULL when visible is. */
int gsb_stereo_pack_inputs(const uint8_t* left, const uint8_t* right, int32_t width, int32_t height, float* out, void* stream);
int gsb_stereo_disparities(const float* flow_lr, const float* flow_rl, int32_t width, int32_t height, float sign, float* disp_lr,
                           float* disp_rl, void* stream);
int gsb_stereo_occlusion_depth(const float* disp_lr, const float* disp_rl, int32_t width, int32_t height, int64_t rl_stride,
                               double threshold, float depth_numerator, uint8_t* visible, float* depth, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GS2MESH_B200_H_ */
