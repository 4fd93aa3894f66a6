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
  GSB_ERR_WORKSPACE = 2,  /* caller workspace too small; see gsb_raster_required_instances */
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

/* flags for GsbRasterArgs.flags */
#define GSB_RASTER_EXACT_TILE_CULL 1u /* drop (Gaussian,tile) pairs that provably contribute to no
                                         pixel of the tile; image is bit-identical, num_rendered
                                         shrinks.  Off = reference rectangle binning
                                         (rasterizer_impl.cu:88-107).                          */
#define GSB_RASTER_NO_TMA 2u          /* stage parameters with plain loads (debug / A-B only)  */
#define GSB_RASTER_DEBUG_SYNC 4u      /* synchronise + check after every stage, like debug=True
                                         (auxiliary.h:166-173)                                 */
#define GSB_RASTER_CUB_SORT 8u        /* validation only: the reference's pipeline shape (P-sized scan,
                                         cub::DeviceRadixSort on tile|depth keys, host read of the
                                         instance count) instead of the in-library depth-presort +
                                         stable tile split                                      */
#define GSB_RASTER_FAST_EXP 32u       /* blend with ex2.approx(power*log2e) instead of full-precision
                                         expf: ~2e-7 relative on alpha (parity budget is 1e-4)   */
/* A/B overrides of the library defaults, for tests and profiling (0 in a field = library default, which the
 * environment variables GSB_RENDER_IMPL / GSB_PRE_SH may also change):
 *   bits 8..10  blend kernel: 4 dual (per-warp compacted hit lists, 8x8 pixels per warp, the reference's exponent
 *               expression), 5 table (dual with per-column / per-row exponent tables, packed f32x2 and predicated
 *               accumulation; default, needs GSB_RASTER_FAST_EXP -- without it the dual kernel runs); 1..3 (variants
 *               removed in round 2) select dual
 *   bits 12..13 SH staging of full-degree blocks: 1 scalar reads, 2 16-byte reads (default), 3 per-lane bulk copies
 *               into padded slots + 16-byte reads
 * dual produces the reference's transmittance bit for bit when GSB_RASTER_FAST_EXP is off; table rounds the exponent
 * differently (~1e-6 relative on alpha). */
#define GSB_RASTER_RENDER_IMPL(n) (((uint32_t)(n) & 7u) << 8)
#define GSB_RASTER_SH_MODE(n) (((uint32_t)(n) & 3u) << 12)
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
     [0] = instances actually binned, [1] = reference-equivalent count (sum of tile rectangles,
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
 * returns GSB_ERR_WORKSPACE and gsb_raster_required_instances() tells how many are needed
 * (outputs are then undefined).  Without GSB_RASTER_ASYNC the call waits for the stream ONCE, at
 * the end of the frame, to be able to report that; the reference blocks in the middle of the
 * frame instead (rasterizer_impl.cu:281).  With GSB_RASTER_ASYNC nothing waits. */
int gsb_raster_forward(const GsbRasterArgs* args, void* stream);
int64_t gsb_raster_required_instances(void);

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
 * Lattice indices must lie in [-2^20, 2^20) per axis.  When the pool is exhausted further bricks are dropped and counted
 * (gsb_tsdf_last_stats); the caller grows the pool and integrates again. */
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
                                          [4] pool slots in use, [5] bricks dropped since creation     */
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

/* volume.integrate(rgbd, intrinsic, extrinsic): depth = prepared float depth [H,W] (device),
 * rgb = uint8 [H,W,3] (device) or NULL, extrinsic_w2c = row-major double[16] on the HOST
 * (what tsdf_utils.py:107 passes: inv(left_camera['extrinsic'])). */
int gsb_tsdf_integrate(GsbVolume* vol, const float* depth, const uint8_t* rgb, int32_t width, int32_t height, double fx,
                       double fy, double cx, double cy, const double* extrinsic_w2c, void* stream);

/* Block discovery only (T1): opens the bricks the frame would touch without updating any voxel.  Lets a caller that must
 * never lose a brick (the Open3D-shaped facade) check gsb_tsdf_last_stats and grow the pool BEFORE integrating. */
int gsb_tsdf_touch(GsbVolume* vol, const float* depth, int32_t width, int32_t height, double fx, double fy, double cx, double cy,
                   const double* extrinsic_w2c, void* stream);

/* (mean, weight) <-> (sum, weight) of every pool slot in use / of the listed pool slots (device uint32[n_bricks]);
 * to_sums != 0: (mean,w) -> (sum,w).  Building blocks of the cross-rank merge below. */
int gsb_tsdf_to_sums(GsbVolume* vol, void* stream);
int gsb_tsdf_from_sums(GsbVolume* vol, void* stream);
int gsb_tsdf_sums_bricks(GsbVolume* vol, int to_sums, const uint32_t* bricks, uint32_t n_bricks, void* stream);

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
 * integrate, [1] bricks it had to drop (pool exhausted / index out of range), [2] frame id, [3] pool slots in use,
 * [4] bricks dropped since creation. */
int gsb_tsdf_last_stats(const GsbVolume* vol, uint32_t* out, void* stream);

/* ------------------------------------------------------------------------------------------
 * Multi-GPU merge of view-sharded volumes (SURVEY.md 8(b) seam 2, 8(e)): ONE call per rank,
 *     gsb_tsdf_reduce(vol, comm, root, scratch, scratch_bytes, stream)
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
/* Returns GSB_ERR_WORKSPACE when `scratch` cannot hold the packed union (known only after the index exchange);
 * gsb_tsdf_reduce_required_bytes() then tells the size to retry with.  The required size is the same on every rank, so
 * ranks that pass equally sized scratch blocks take the same decision (a collective must not be entered by some ranks
 * only); a retry repeats the cheap index exchange.  root >= 0: ncclReduce to `root` (only its volume is changed);
 * root < 0: ncclAllReduce (every rank ends with the merged volume). */
int gsb_tsdf_reduce(GsbVolume* vol, void* nccl_comm, int nranks, int rank, int root, void* scratch, size_t scratch_bytes,
                    void* stream);
size_t gsb_tsdf_reduce_required_bytes(void);
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
 * unique edges.
 *   gsb_mesh_count    tri_counts[b]  = triangles produced by brick b
 *   gsb_mesh_emit     edge_keys[3*t..3*t+2] for every triangle, brick b writing from tri_offsets[b]
 *   gsb_mesh_vertices xyz (fp64, Open3D's interpolation) and rgb in [0,1] (or NULL) of n unique keys
 *   gsb_mesh_vertex_normals area-weighted vertex normals (fp64 [n_vertices,3]) of an indexed mesh */
int gsb_mesh_count(const GsbVolume* vol, const int32_t* window, const uint32_t* bricks, uint32_t n_bricks, uint32_t* tri_counts,
                   void* stream);
int gsb_mesh_emit(const GsbVolume* vol, const int32_t* window, const uint32_t* bricks, uint32_t n_bricks, const int64_t* tri_offsets,
                  int64_t* edge_keys, void* stream);
int gsb_mesh_vertices(const GsbVolume* vol, const int32_t* window, const int64_t* keys, int64_t n, double* xyz, float* rgb,
                      void* stream);
int gsb_mesh_vertex_normals(const double* xyz, int64_t n_vertices, const int64_t* triangles, int64_t n_triangles, double* normals,
                            void* stream);

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
  int32_t dims[3];          /* cells per axis; dims[0]*dims[1]*dims[2] < 2^31           */
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
 * until the nearest point is found. */
int gsb_eval_nearest(const GsbPointGrid* grid, const double* queries, int64_t n_queries, double max_dist, double* dist,
                     int64_t* index, void* stream);
/* Greedy radius downsampling of the grid's points in index order (eval.py:88-93): keep[p] = 1 iff no earlier kept point q
 * has ((dx*dx)+dy*dy)+dz*dz <= radius*radius (sklearn radius_neighbors, inclusive).  Needs grid->cell > radius.
 * Runs rounds of the parallel greedy rule and reads the undecided count every 4 rounds: SYNCHRONISES the stream.
 * keep: device uint8[n_points]; counters: device uint32[4] scratch; host_undecided: pinned host uint32[1];
 * rounds (may be NULL) receives the number of rounds run. */
int gsb_eval_radius_downsample(const GsbPointGrid* grid, double radius, uint8_t* keep, uint32_t* counters,
                               uint32_t* host_undecided, int32_t* rounds, void* stream);

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

#ifdef __cplusplus
}
#endif
#endif /* GS2MESH_B200_H_ */
